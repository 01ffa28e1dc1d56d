"""ResNeXt / Wide ResNet on CPU: torchvision parity (state_dict, parameter counts, forward and gradients) and the
grouped-conv plumbing that needs no GPU."""
import pytest
import torch
import torchvision

from distributeddeeplearning_b200 import models, ops
from distributeddeeplearning_b200.models.layers import Conv2d
from distributeddeeplearning_b200.ops import native
from distributeddeeplearning_b200.ops.functional import is_stem_weight

PARAMS = {"resnext50_32x4d": 25_028_904, "resnext101_32x8d": 88_791_336, "resnext101_64x4d": 83_455_272,
          "wide_resnet50_2": 68_883_240, "wide_resnet101_2": 126_886_696}


@pytest.mark.parametrize("name", sorted(PARAMS))
def test_state_dict_and_param_count_match_torchvision(name):
    m = models.get_model(name)
    tv = getattr(torchvision.models, name)()
    assert {k: tuple(v.shape) for k, v in m.state_dict().items()} == {k: tuple(v.shape) for k, v in tv.state_dict().items()}
    n = sum(p.numel() for p in m.parameters())
    assert n == sum(p.numel() for p in tv.parameters()) == PARAMS[name]


def test_resnext50_forward_backward_equals_torchvision():
    torch.manual_seed(0)
    m, tv = models.get_model("resnext50_32x4d"), torchvision.models.resnext50_32x4d()
    m.load_state_dict(tv.state_dict())
    tv = tv.double()          # small batches make BN backward ill-conditioned: compare against float64
    m.train(), tv.train()
    x = torch.randn(4, 3, 96, 96)
    y = torch.tensor([1, 7, 3, 9])
    o1, o2 = m(x), tv(x.double())
    assert torch.allclose(o1.double(), o2, atol=5e-4, rtol=1e-3)
    ops.softmax_cross_entropy(o1, y).backward()
    torch.nn.functional.cross_entropy(o2, y).backward()
    g1, g2 = dict(m.named_parameters()), dict(tv.named_parameters())
    for k in ("conv1.weight", "layer1.0.conv2.weight", "layer2.0.conv2.weight", "layer3.1.conv2.weight",
              "layer4.2.conv2.weight", "layer2.0.downsample.0.weight", "layer1.0.bn2.weight", "fc.bias"):
        err = float((g1[k].grad.double() - g2[k].grad).norm() / g2[k].grad.norm())
        # a wrong group mapping is O(1); a ReLU / max decision near zero in the 3x3 layer4 maps flipping under fp32
        # summation order moves every gradient below it by a few percent
        assert err < 5e-2, (k, err)
    assert tuple(g1["layer1.0.conv2.weight"].grad.shape) == (128, 4, 3, 3)
    for k in ("bn1", "layer1.0.bn2", "layer3.0.bn2", "layer4.2.bn3"):
        a, b = m.get_submodule(k), tv.get_submodule(k)
        assert torch.allclose(a.running_mean.double(), b.running_mean, atol=1e-5), k
        assert torch.allclose(a.running_var.double(), b.running_var, atol=1e-5, rtol=1e-4), k


def test_grouped_conv2d_loads_nn_conv2d_state_dict():
    ref = torch.nn.Conv2d(256, 256, 3, 2, 1, groups=32, bias=False)
    c = Conv2d(256, 256, 3, 2, 1, groups=32)
    assert tuple(c.weight.shape) == (256, 8, 3, 3)
    c.load_state_dict(ref.state_dict())
    assert c.weight.is_contiguous(memory_format=torch.channels_last)
    assert torch.equal(c.weight, ref.weight)
    assert set(c.state_dict()) == set(ref.state_dict())
    x = torch.randn(1, 256, 9, 9)
    assert torch.allclose(c(x), ref(x), atol=1e-5, rtol=1e-5)


def test_grouped_weight_is_not_a_stem_weight():
    c = Conv2d(128, 128, 3, 1, 1, groups=32)
    assert tuple(c.weight.shape) == (128, 4, 3, 3)
    assert not is_stem_weight(c.weight)
    assert not is_stem_weight(torch.empty(128, 4, 3, 3), groups=32)
    assert is_stem_weight(Conv2d(3, 64, 7, 2, 3).weight)


def test_supports_grouped_predicate():
    for c, g in ((128, 32), (256, 32), (1024, 32), (2048, 64), (512, 64), (128, 2)):
        assert native.supports_grouped(c, c, g), (c, g)
    assert not native.supports_grouped(128, 256, 32)      # Cin != Cout
    assert not native.supports_grouped(96, 96, 3)         # not a multiple of 64
    assert not native.supports_grouped(128, 128, 64)      # group width 2
    assert not native.supports_grouped(128, 128, 128)     # depthwise
    assert not native.supports_grouped(384, 384, 4)       # group width 96 does not divide 64
    assert not models.get_model("resnet50").layer1[0].conv2.groups > 1
