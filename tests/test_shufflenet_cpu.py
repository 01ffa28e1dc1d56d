"""ShuffleNetV2 x0.5 / x1.0 / x1.5 / x2.0 on CPU: torchvision parity (state_dict, parameter counts, initialisation,
eval logits and train-mode gradients in float64), the unit composite against torchvision's ``InvertedResidual`` at both
strides (the 58- and 122-wide units included), the builder arguments, and the compiled shuffle kernels (ptxas)."""
import math
import os
import re
import shutil
import subprocess

import pytest
import torch
import torchvision
from torchvision.models.shufflenetv2 import InvertedResidual as TvUnit

from distributeddeeplearning_b200 import _ext, models
from distributeddeeplearning_b200.models.shufflenetv2 import InvertedResidual
from distributeddeeplearning_b200.ops.shufflenet import shuffle_unit_composite

NAMES = ["shufflenet_v2_x0_5", "shufflenet_v2_x1_0", "shufflenet_v2_x1_5", "shufflenet_v2_x2_0"]
PARAMS = {"shufflenet_v2_x0_5": 1_366_792, "shufflenet_v2_x1_0": 2_278_604, "shufflenet_v2_x1_5": 3_503_624,
          "shufflenet_v2_x2_0": 7_393_996}


def _copy_from(m, tv):
    m.load_state_dict(tv.state_dict())


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


@pytest.mark.parametrize("name", NAMES)
def test_state_dict_and_parameter_count_match_torchvision(name):
    m = models.get_model(name)
    tv = getattr(torchvision.models, name)()
    sd, tsd = m.state_dict(), tv.state_dict()
    assert list(sd) == list(tsd)
    assert [(tuple(v.shape), v.dtype) for v in sd.values()] == [(tuple(v.shape), v.dtype) for v in tsd.values()]
    assert sum(p.numel() for p in m.parameters()) == sum(p.numel() for p in tv.parameters()) == PARAMS[name]
    for k in ("conv1.0.weight", "conv1.1.running_var", "stage2.0.branch1.2.weight", "stage2.1.branch2.6.bias",
              "conv5.1.weight", "fc.bias"):
        assert k in sd
    assert not any(k.startswith("stage2.1.branch1") for k in sd)       # the empty branch1 of stride-1 units
    assert models.input_size(name) == models.input_size(m) == 224


def test_builder_arguments():
    assert models.get_model("shufflenet_v2_x1_0", num_classes=10).fc.out_features == 10
    with pytest.raises(ValueError):
        models.get_model("shufflenet_v2_x1_0", dropout=0.1)


def test_initialisation_matches_torchvision_defaults():
    torch.manual_seed(0)
    m = models.get_model("shufflenet_v2_x1_0")
    for name, p in m.named_parameters():
        if p.dim() == 4:                          # kaiming_uniform(a=sqrt(5)): U(-1/sqrt(fan_in), 1/sqrt(fan_in))
            bound = 1 / math.sqrt(p[0].numel())
            assert p.abs().max() <= bound + 1e-7, name
            assert abs(p.std().item() - bound / math.sqrt(3)) < 0.1 * bound / math.sqrt(3) + 5e-3 * (p.numel() < 500), name
        elif name.endswith("weight") and p.dim() == 1:
            assert torch.equal(p, torch.ones_like(p)), name
        elif p.dim() == 1 and not name.startswith("fc"):
            assert torch.equal(p, torch.zeros_like(p)), name
    bound = 1 / math.sqrt(1024)
    assert m.fc.weight.abs().max() <= bound and m.fc.bias.abs().max() <= bound
    for name, b in m.named_buffers():
        if name.endswith("running_mean"):
            assert torch.equal(b, torch.zeros_like(b))
        elif name.endswith("running_var"):
            assert torch.equal(b, torch.ones_like(b))


@pytest.mark.parametrize("name", ["shufflenet_v2_x0_5", "shufflenet_v2_x1_0"])
def test_eval_logits_match_torchvision_float64(name):
    torch.manual_seed(1)
    tv = getattr(torchvision.models, name)()
    _randomize(tv, 7)
    m = models.get_model(name)
    _copy_from(m, tv)
    m.eval(), tv.double().eval()
    x = torch.randn(2, 3, 224, 224)
    with torch.no_grad():
        got, ref = m(x).double(), tv(x.double())
    assert got.shape == (2, 1000)
    assert float((got - ref).abs().max()) <= 1e-4 * float(ref.abs().max()) + 1e-9


def test_train_gradients_match_torchvision_float64():
    torch.manual_seed(2)
    tv = torchvision.models.shufflenet_v2_x1_0()
    _randomize(tv, 3)
    m = models.get_model("shufflenet_v2_x1_0")
    _copy_from(m, tv)
    m.train(), tv.double().train()          # small batches make BN backward ill-conditioned: compare against float64
    x = torch.randn(4, 3, 96, 96)
    y = torch.tensor([1, 5, 9, 3])
    o1, o2 = m(x), tv(x.double())
    assert torch.allclose(o1.double(), o2, atol=5e-4, rtol=1e-3)
    torch.nn.functional.cross_entropy(o1, y).backward()
    torch.nn.functional.cross_entropy(o2, y).backward()
    g1 = dict(m.named_parameters())
    for k, p in tv.named_parameters():
        err = float((g1[k].grad.double() - p.grad).norm() / max(float(p.grad.norm()), 1e-4))
        assert err < 5e-2, (k, err)
    tb = dict(tv.named_buffers())
    for k, b in m.named_buffers():
        if "running" in k:
            assert torch.allclose(b.double(), tb[k], atol=1e-5, rtol=1e-4), k


def _tv_params(u, stride):
    """The unit's tensors for the composite, with copies of the running statistics."""
    def bn(b):
        return (b.weight, b.bias, b.running_mean.clone(), b.running_var.clone(), b.eps, b.momentum)

    b2 = (u.branch2[0].weight, bn(u.branch2[1]), u.branch2[3].weight, bn(u.branch2[4]), u.branch2[5].weight,
          bn(u.branch2[6]))
    b1 = None if stride == 1 else (u.branch1[0].weight, bn(u.branch1[1]), u.branch1[2].weight, bn(u.branch1[3]))
    return b2, b1


@pytest.mark.parametrize("inp,oup,stride,hw", [(24, 116, 2, 14), (116, 116, 1, 9), (244, 244, 1, 7), (24, 244, 2, 10),
                                               (232, 464, 2, 8), (48, 48, 1, 6)])
@pytest.mark.parametrize("training", [True, False])
def test_unit_composite_matches_torchvision(inp, oup, stride, hw, training):
    torch.manual_seed(inp + oup + stride)
    tv = TvUnit(inp, oup, stride).double()
    _randomize(tv, inp)
    tv.train(training)
    b2, b1 = _tv_params(tv, stride)
    x = torch.randn(2, inp, hw, hw, dtype=torch.float64, requires_grad=True)
    ref = tv(x)
    xc = x.detach().clone().requires_grad_(True)
    got = shuffle_unit_composite(xc, b2, b1, training)
    assert torch.allclose(got, ref, rtol=1e-10, atol=1e-10)
    bns = [b2[1], b2[3], b2[5]] + ([b1[1], b1[3]] if b1 is not None else [])
    tv_bns = [tv.branch2[i] for i in (1, 4, 6)] + ([tv.branch1[i] for i in (1, 3)] if b1 is not None else [])
    for ours, theirs in zip(bns, tv_bns):
        assert torch.allclose(ours[2], theirs.running_mean, rtol=1e-12, atol=1e-14)
        assert torch.allclose(ours[3], theirs.running_var, rtol=1e-12, atol=1e-14)
    ref.backward(torch.ones_like(ref))
    got.backward(torch.ones_like(got))
    assert torch.allclose(xc.grad, x.grad, rtol=1e-9, atol=1e-10)


def test_unit_module_runs_the_composite_on_cpu():
    torch.manual_seed(4)
    ours, tv = InvertedResidual(58 * 2, 58 * 2, 1, whole_output=True), TvUnit(116, 116, 1)
    _randomize(tv, 5)
    ours.load_state_dict(tv.state_dict())
    x = torch.randn(2, 116, 7, 7)
    assert torch.allclose(ours(x), tv(x), rtol=1e-5, atol=1e-5)


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
def test_shuffle_kernels_compile_without_spills():
    k = _ptxas("shufflenet.cu")
    assert sorted(k) == sorted(["shuffle_fwd_kernel<true, true>", "shuffle_fwd_kernel<true, false>",
                                "shuffle_fwd_kernel<false, true>", "shuffle_fwd_kernel<false, false>",
                                "shuffle_bwd_reduce_kernel<true>", "shuffle_bwd_reduce_kernel<false>",
                                "shuffle_bwd_apply_kernel<true>", "shuffle_bwd_apply_kernel<false>"]), sorted(k)
    for name, (regs, st, ld) in k.items():
        assert st == 0 and ld == 0 and regs <= 128, (name, regs, st, ld)        # __launch_bounds__(256): 2 CTAs / SM
    se = _ptxas("squeeze_excite_sigmoid.cu")
    for name in ("pad_cols_kernel", "fold_cols_kernel"):
        assert name in se and se[name][1:] == [0, 0], (name, se.get(name))
