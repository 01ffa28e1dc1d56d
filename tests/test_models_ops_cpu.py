"""Model zoo + op composites on CPU: torchvision parity (state_dict keys, forward, gradients)."""
import pytest
import torch
import torchvision

from distributeddeeplearning_b200 import models, ops
from distributeddeeplearning_b200.ops import native


@pytest.mark.parametrize("name", ["resnet18", "resnet50", "resnet101", "resnet152", "vgg16", "vgg11_bn", "alexnet",
                                  "inception_v3", "densenet121", "densenet161", "squeezenet1_0", "squeezenet1_1"])
def test_state_dict_matches_torchvision(name):
    m = models.get_model(name)
    kw = {"init_weights": False} if "inception" in name else {}
    tv = getattr(torchvision.models, name)(**kw)
    a = {k: tuple(v.shape) for k, v in m.state_dict().items()}
    b = {k: tuple(v.shape) for k, v in tv.state_dict().items()}
    assert a == b


def test_param_counts_match_survey():
    # SURVEY.md 2.7 [measured-here]
    assert sum(p.numel() for p in models.get_model("resnet50").parameters()) == 25_557_032
    assert sum(p.numel() for p in models.get_model("vgg16").parameters()) == 138_357_544
    assert sum(p.numel() for p in models.get_model("alexnet").parameters()) == 61_100_840
    assert sum(p.numel() for p in models.get_model("inception_v3").parameters()) == 27_161_264
    assert len(list(models.get_model("resnet50").parameters())) == 161


def test_resnet18_forward_backward_equals_torchvision():
    torch.manual_seed(0)
    m, tv = models.get_model("resnet18"), torchvision.models.resnet18()
    m.load_state_dict(tv.state_dict())
    m.train(), tv.train()
    x = torch.randn(2, 3, 64, 64)
    y = torch.tensor([1, 7])
    o1, o2 = m(x), tv(x)
    assert torch.allclose(o1, o2, atol=1e-4, rtol=1e-4)
    ops.softmax_cross_entropy(o1, y).backward()
    torch.nn.functional.cross_entropy(o2, y).backward()
    g1, g2 = dict(m.named_parameters()), dict(tv.named_parameters())
    for k in ("conv1.weight", "layer2.0.downsample.0.weight", "fc.bias", "layer4.1.bn2.weight"):
        assert torch.allclose(g1[k].grad, g2[k].grad, atol=1e-4, rtol=1e-3), k
    # running statistics were updated identically
    assert torch.allclose(m.bn1.running_mean, tv.bn1.running_mean, atol=1e-5)


def test_vgg_alexnet_forward_equal_torchvision_eval():
    torch.manual_seed(0)
    for name in ("alexnet", "vgg11"):
        m, tv = models.get_model(name), getattr(torchvision.models, name)()
        m.load_state_dict(tv.state_dict())
        m.eval(), tv.eval()
        x = torch.randn(1, 3, 224, 224)
        with torch.no_grad():
            assert torch.allclose(m(x), tv(x), atol=1e-3, rtol=1e-3), name


def test_densenet_squeezenet_match_torchvision():
    torch.manual_seed(0)
    for name in ("densenet121", "squeezenet1_1"):
        m, tv = models.get_model(name), getattr(torchvision.models, name)()
        m.load_state_dict(tv.state_dict())
        m.eval(), tv.eval()
        x = torch.randn(1, 3, 96, 96)
        with torch.no_grad():
            assert torch.allclose(m(x), tv(x), atol=1e-4, rtol=1e-3), name
    # pre-activation BN + concat path in train mode: gradients equal torchvision's
    m, tv = models.get_model("densenet121"), torchvision.models.densenet121()
    m.load_state_dict(tv.state_dict())
    m.train(), tv.train()
    x, y = torch.randn(2, 3, 64, 64), torch.tensor([3, 5])
    o1, o2 = m(x), tv(x)
    assert torch.allclose(o1, o2, atol=1e-4, rtol=1e-3)
    ops.softmax_cross_entropy(o1, y).backward()
    torch.nn.functional.cross_entropy(o2, y).backward()
    g1, g2 = dict(m.named_parameters()), dict(tv.named_parameters())
    for k in ("features.conv0.weight", "features.denseblock2.denselayer3.conv2.weight", "features.transition1.conv.weight",
              "features.norm5.weight", "classifier.bias"):
        ref = g2[k].grad
        assert (g1[k].grad - ref).abs().max() <= 1e-2 * ref.abs().max() + 1e-5, k   # 121 BN layers, batch 2: fp32 order noise


def test_concat_channels_composite():
    a, b = torch.randn(2, 8, 3, 3, requires_grad=True), torch.randn(2, 16, 3, 3, requires_grad=True)
    out = ops.concat_channels([a, b])
    assert out.shape == (2, 24, 3, 3)
    out.sum().backward()
    assert torch.equal(a.grad, torch.ones_like(a)) and torch.equal(b.grad, torch.ones_like(b))


def test_inception_returns_aux_in_train_mode():
    m = models.get_model("inception_v3")
    assert models.input_size(m) == 299 and models.input_size("inception_v3") == 299
    m.train()
    out = m(torch.randn(2, 3, 299, 299))
    assert isinstance(out, tuple) and out[0].shape == (2, 1000) and out[1].shape == (2, 1000)
    m.eval()
    with torch.no_grad():
        assert m(torch.randn(1, 3, 299, 299)).shape == (1, 1000)


def test_registry():
    assert "resnet50" in models.available_models() and "vgg16" in models.available_models()
    with pytest.raises(ValueError):
        models.get_model("nope")
    with pytest.raises(ValueError):
        models.get_model("resnet50", pretrained=True)


def test_topk_and_xent_composites():
    logits = torch.tensor([[5.0, 1.0, 0.0, 0.0, 0.0, 0.0, 9.0], [0.0, 3.0, 2.0, 1.0, 0.5, 0.4, 9.0]])
    labels = torch.tensor([0, 5])
    # last column is padding: classes=6 must ignore it
    corr = ops.topk_correct(logits, labels, classes=6)
    assert corr.tolist() == [1, 2]
    loss = ops.softmax_cross_entropy(logits, labels, classes=6)
    assert loss.item() == pytest.approx(torch.nn.functional.cross_entropy(logits[:, :6], labels).item())


def test_stem_geometry_and_support_matrix():
    assert native.stem_geometry(7, 7) == (8, 2, 4, 8)       # ResNet stem: 4 k-blocks of 2 rows x 8 taps x 4 ch
    assert native.stem_geometry(11, 11) == (16, 1, 11, 11)  # AlexNet
    assert native.stem_geometry(3, 3) == (4, 4, 1, 4)       # VGG
    # any channel count that is a multiple of 8 (Inception's 80 -> 192), or an NHWC4 stem
    assert native.supports_conv(64, 256) and native.supports_conv(3, 64) and native.supports_conv(80, 192)
    assert not native.supports_conv(20, 64) and not native.supports_conv(64, 1000 + 4)
    assert native.bn_supported(2048) and native.bn_supported(64) and native.bn_supported(80) and not native.bn_supported(12)
    assert native.conv_out_hw(224, 224, (7, 7), 2, 3) == (112, 112)
    assert native.conv_out_hw(17, 17, (1, 7), 1, (0, 3)) == (17, 17)       # asymmetric Inception kernels


def test_stem_tma_geometry_and_padding_rules():
    # ResNet stem 7x7/2 pad 3 on 224: 2 filter rows per k-block -> 2-row interleave, 230x230 padded image
    assert native.stem_tma_geometry(224, 224, (7, 7), 2, 3) == (230, 230, 2)
    # AlexNet 11x11/4 pad 2: one row per k-block, width padded so the last window's 16 taps stay in bounds (even width)
    hp, wp, g = native.stem_tma_geometry(224, 224, (11, 11), 4, 2)
    assert g == 1 and wp % 2 == 0 and wp >= 4 * 54 + 16 and hp >= 228
    # 3x3/1 (VGG): 4-row interleave makes the per-pixel step 32 bytes -> TMA-eligible
    assert native.stem_tma_geometry(224, 224, (3, 3), 1, 1)[2] == 4
    # 11x11 stride 1 would need an 8-byte column step: gather path
    assert native.stem_tma_geometry(64, 64, (11, 11), 1, 5) is None
    assert native._pad2(3) == (3, 3) and native._pad2((0, 3)) == (0, 3)


def test_graphed_step_not_applicable_on_cpu_and_dropout_detection():
    from distributeddeeplearning_b200.workloads.graph_step import GraphedStep, model_has_dropout

    m = models.get_model("resnet18")
    opt = torch.optim.SGD(m.parameters(), lr=0.1)
    assert not GraphedStep.applicable(m, opt, torch.zeros(1, 3, 8, 8))
    assert not model_has_dropout(m) and model_has_dropout(models.get_model("alexnet"))
    ops.advance_dropout_step()                                     # no GPU dropout ran: a no-op
    g = GraphedStep(lambda a: a + 1, opt)
    assert not g.matches((torch.zeros(2),))
    assert torch.equal(g(torch.zeros(2)), torch.ones(2))          # falls back to the eager function


def test_batch_norm_act_composite_matches_torch():
    x = torch.randn(4, 8, 5, 5, requires_grad=True)
    g, b = torch.rand(8) + 0.5, torch.randn(8)
    rm, rv = torch.zeros(8), torch.ones(8)
    z = ops.batch_norm_act(x, g, b, rm, rv, 1e-5, 0.1, True, True)
    ref = torch.relu(torch.nn.functional.batch_norm(x, torch.zeros(8), torch.ones(8), g, b, True, 0.1, 1e-5))
    assert torch.allclose(z, ref, atol=1e-5)


def test_bn3_handoff_hands_sums_only_to_the_unmodified_gradient():
    """A block takes the BN3 sums of the next block's dgrad only for the very tensor that dgrad returned, unmodified,
    and only once."""
    from distributeddeeplearning_b200.ops.blocks import _Bn3Handoff

    d = torch.randn(2, 16, 3, 3).contiguous(memory_format=torch.channels_last)

    def armed():
        h = _Bn3Handoff()
        h.bn, h.sums, h.dx, h.version = ("y", "save", "gamma", "beta", "mask"), torch.randn(2, 16), d, d._version
        return h

    h = armed()
    sums = h.sums
    assert h.pre_reduced(d) is sums
    assert h.bn is None and h.sums is None and h.dx is None       # cleared: the next call finds nothing
    assert h.pre_reduced(d) is None
    assert armed().pre_reduced(d.clone()) is None                   # same values, different storage
    assert armed().pre_reduced(d[:1]) is None                       # same storage start, different shape
    h = armed()
    d.mul_(2.0)                                                     # modified in place: the version moved on
    assert h.pre_reduced(d) is None
    assert armed().pre_reduced(d) is not None                       # re-armed at the current version
    assert _Bn3Handoff().pre_reduced(d) is None                     # never armed
