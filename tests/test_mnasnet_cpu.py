"""MNASNet 0.5 / 0.75 / 1.0 / 1.3 on CPU: torchvision parity (state_dict, parameter counts, checkpoints loading strictly
in both directions, which at alpha != 1.0 needs the version-2 metadata, initialisation, eval logits and train-mode
gradients in float64) and the builder arguments."""
import math

import pytest
import torch
import torchvision

from distributeddeeplearning_b200 import models
from distributeddeeplearning_b200.models.mnasnet import _get_depths

NAMES = ["mnasnet0_5", "mnasnet0_75", "mnasnet1_0", "mnasnet1_3"]
PARAMS = {"mnasnet0_5": 2_218_512, "mnasnet0_75": 3_170_208, "mnasnet1_0": 4_383_312, "mnasnet1_3": 6_282_256}


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
    assert sd._metadata[""]["version"] == 2
    assert models.input_size(name) == models.input_size(m) == 224
    # checkpoints load strictly in both directions (torchvision reads the root version: 1 would mean the old stem)
    tv.load_state_dict(m.state_dict(), strict=True)
    m.load_state_dict(tv.state_dict(), strict=True)
    for k, v in tv.state_dict().items():
        assert torch.equal(v, sd[k]), k


def test_depths():
    assert _get_depths(0.5) == [16, 8, 16, 24, 40, 48, 96, 160]
    assert _get_depths(1.3) == [40, 24, 32, 56, 104, 128, 248, 416]
    for a in (0.5, 0.75, 1.0, 1.3):
        assert all(d % 8 == 0 for d in _get_depths(a))


def test_builder_arguments():
    m = models.get_model("mnasnet1_0", num_classes=10, dropout=0.5)
    assert m.classifier[1].out_features == 10 and m.classifier[0].p == 0.5
    with pytest.raises(TypeError):
        models.get_model("mnasnet1_0", alpha=2.0)


def test_initialisation_matches_torchvision():
    torch.manual_seed(0)
    m = models.get_model("mnasnet1_0")
    for name, mod in m.named_modules():
        if hasattr(mod, "running_var"):
            assert torch.equal(mod.weight, torch.ones_like(mod.weight)) and torch.equal(mod.bias, torch.zeros_like(mod.bias))
            assert mod.momentum == pytest.approx(1 - 0.9997) and mod.eps == 1e-5
    for name, p in m.named_parameters():
        if p.dim() == 4 and p.numel() > 2000:          # kaiming_normal fan_out, relu: std = sqrt(2 / fan_out)
            std = math.sqrt(2.0 / (p.shape[0] * p.shape[2] * p.shape[3]))
            assert abs(p.std().item() - std) < 0.1 * std, name
    fc = m.classifier[1]                               # kaiming_uniform fan_out, "sigmoid" gain 1: U(+-sqrt(3 / fan_out))
    bound = math.sqrt(3.0 / fc.weight.shape[0])
    assert fc.weight.abs().max() <= bound and fc.weight.abs().max() > 0.9 * bound
    assert torch.equal(fc.bias, torch.zeros_like(fc.bias))


@pytest.mark.parametrize("name", ["mnasnet0_5", "mnasnet1_3"])
def test_eval_logits_match_torchvision_float64(name):
    torch.manual_seed(1)
    tv = getattr(torchvision.models, name)()
    _randomize(tv, 7)
    m = models.get_model(name)
    m.load_state_dict(tv.state_dict())
    m.eval(), tv.double().eval()
    x = torch.randn(2, 3, 224, 224)
    with torch.no_grad():
        got, ref = m(x).double(), tv(x.double())
    assert got.shape == (2, 1000)
    assert float((got - ref).abs().max()) <= 1e-4 * float(ref.abs().max()) + 1e-9


def test_train_gradients_match_torchvision_float64():
    torch.manual_seed(2)
    tv = torchvision.models.mnasnet1_0(dropout=0.0)
    _randomize(tv, 3)
    m = models.get_model("mnasnet1_0", dropout=0.0)
    m.load_state_dict(tv.state_dict())
    m.train(), tv.double().train()
    x = torch.randn(8, 3, 96, 96)
    y = torch.tensor([1, 5, 9, 3, 0, 7, 2, 8])
    o1, o2 = m(x), tv(x.double())
    assert torch.allclose(o1.double(), o2, atol=5e-4, rtol=1e-3)
    torch.nn.functional.cross_entropy(o1, y).backward()
    torch.nn.functional.cross_entropy(o2, y).backward()
    g1 = dict(m.named_parameters())
    for k, p in tv.named_parameters():
        # floor: the stem's last BN has no activation and feeds a train-mode conv + BN, which cancels any shift of its
        # input, so the true gradient of layers.7.bias is zero and both sides carry rounding noise only
        err = float((g1[k].grad.double() - p.grad).norm() / max(float(p.grad.norm()), 1e-3))
        assert err < 5e-2, (k, err)
    tb = dict(tv.named_buffers())
    for k, b in m.named_buffers():
        if "running" in k:
            assert torch.allclose(b.double(), tb[k], atol=1e-5, rtol=1e-4), k
