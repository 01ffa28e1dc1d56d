"""Model zoo (same names as ``torchvision.models`` so ``--model <name>`` keeps working).

Parity: the reference resolves ``--model`` with ``getattr(torchvision.models, name)()``
(``pytorch_synthetic_benchmark.py:60``) / ``models.__dict__[model](pretrained=False)``
(``imagenet_pytorch_horovod.py:383``).  North-star zoo: ResNet-50/101/152, VGG-16, Inception-v3,
AlexNet (SURVEY.md 2.7); ResNet-18/34, the other VGG depths, DenseNet and SqueezeNet (the rest of torchvision
0.2.1's families) are here too, and the later ResNet family members of torchvision (ResNeXt-50 32x4d, ResNeXt-101
32x8d / 64x4d, Wide ResNet-50-2 / 101-2), MobileNetV2, MobileNetV3-Large / -Small, EfficientNet-B0 to -B7,
ConvNeXt-Tiny / -Small / -Base / -Large, the Vision Transformers ViT-B/16, -B/32, -L/16 and -L/32, the Swin
Transformers Swin-T, -S and -B, the Swin Transformers V2 Swin-V2-T, -S and -B, MaxViT-T, the RegNets:
RegNetX-400MF, -800MF, -1.6GF, -3.2GF, -8GF, -16GF and -32GF, and RegNetY-400MF, -800MF, -1.6GF, -3.2GF, -8GF, -16GF,
-32GF and -128GF, ShuffleNetV2 x0.5, x1.0, x1.5 and x2.0, GoogLeNet, and MNASNet 0.5, 0.75, 1.0 and 1.3.
"""
from __future__ import annotations

from .alexnet import AlexNet, alexnet  # noqa: F401
from .convnext import ConvNeXt, convnext_base, convnext_large, convnext_small, convnext_tiny  # noqa: F401
from .densenet import DenseNet, densenet121, densenet161, densenet169, densenet201  # noqa: F401
from .efficientnet import (INPUT_SIZE as _EFFICIENTNET_INPUT_SIZE, EfficientNet, efficientnet_b0,  # noqa: F401
                           efficientnet_b1, efficientnet_b2, efficientnet_b3, efficientnet_b4, efficientnet_b5,
                           efficientnet_b6, efficientnet_b7)
from .efficientnet_v2 import (INPUT_SIZE as _EFFICIENTNET_V2_INPUT_SIZE, EfficientNetV2,  # noqa: F401
                              efficientnet_v2_l, efficientnet_v2_m, efficientnet_v2_s)
from .googlenet import GoogLeNet, googlenet  # noqa: F401
from .inception import Inception3, inception_v3  # noqa: F401
from .maxvit import MaxVit, maxvit_t  # noqa: F401
from .mobilenet import MobileNetV2, mobilenet_v2  # noqa: F401
from .mnasnet import MNASNet, mnasnet0_5, mnasnet0_75, mnasnet1_0, mnasnet1_3  # noqa: F401
from .mobilenetv3 import MobileNetV3, mobilenet_v3_large, mobilenet_v3_small  # noqa: F401
from .regnet import (RegNet, regnet_x_1_6gf, regnet_x_3_2gf, regnet_x_8gf, regnet_x_16gf, regnet_x_32gf,  # noqa: F401
                     regnet_x_400mf, regnet_x_800mf, regnet_y_1_6gf, regnet_y_3_2gf, regnet_y_8gf, regnet_y_16gf,
                     regnet_y_32gf, regnet_y_128gf, regnet_y_400mf, regnet_y_800mf)
from .resnet import (ResNet, resnet18, resnet34, resnet50, resnet101, resnet152, resnext50_32x4d,  # noqa: F401
                     resnext101_32x8d, resnext101_64x4d, wide_resnet50_2, wide_resnet101_2)
from .shufflenetv2 import (ShuffleNetV2, shufflenet_v2_x0_5, shufflenet_v2_x1_0,  # noqa: F401
                           shufflenet_v2_x1_5, shufflenet_v2_x2_0)
from .squeezenet import SqueezeNet, squeezenet1_0, squeezenet1_1  # noqa: F401
from .swin import SwinTransformer, swin_b, swin_s, swin_t  # noqa: F401
from .swin_v2 import INPUT_SIZE as _SWIN_V2_INPUT_SIZE, SwinTransformerV2, swin_v2_b, swin_v2_s, swin_v2_t  # noqa: F401
from .vgg import VGG, vgg11, vgg11_bn, vgg13, vgg13_bn, vgg16, vgg16_bn, vgg19, vgg19_bn  # noqa: F401
from .vit import VisionTransformer, vit_b_16, vit_b_32, vit_l_16, vit_l_32  # noqa: F401

_REGISTRY = {
    f.__name__: f
    for f in (alexnet, convnext_tiny, convnext_small, convnext_base, convnext_large, densenet121, densenet161,
              densenet169, densenet201, efficientnet_b0, efficientnet_b1, efficientnet_b2, efficientnet_b3,
              efficientnet_b4, efficientnet_b5, efficientnet_b6, efficientnet_b7, efficientnet_v2_s,
              efficientnet_v2_m, efficientnet_v2_l,
              squeezenet1_0, squeezenet1_1, inception_v3, mobilenet_v2,
              mobilenet_v3_large, mobilenet_v3_small, resnet18, resnet34, resnet50, resnet101, resnet152,
              resnext50_32x4d, resnext101_32x8d, resnext101_64x4d, wide_resnet50_2, wide_resnet101_2, vgg11, vgg11_bn, vgg13,
              vgg13_bn, vgg16, vgg16_bn, vgg19, vgg19_bn, vit_b_16, vit_b_32, vit_l_16, vit_l_32, swin_t, swin_s, swin_b,
              swin_v2_t, swin_v2_s, swin_v2_b, maxvit_t, regnet_x_400mf, regnet_x_800mf, regnet_x_1_6gf,
              regnet_x_3_2gf, regnet_x_8gf, regnet_x_16gf, regnet_x_32gf, regnet_y_400mf, regnet_y_800mf,
              regnet_y_1_6gf, regnet_y_3_2gf, regnet_y_8gf, regnet_y_16gf, regnet_y_32gf, regnet_y_128gf,
              shufflenet_v2_x0_5, shufflenet_v2_x1_0, shufflenet_v2_x1_5, shufflenet_v2_x2_0, googlenet, mnasnet0_5,
              mnasnet0_75, mnasnet1_0, mnasnet1_3)
}


def available_models():
    return sorted(_REGISTRY)


def get_model(name: str, **kw):
    """Build a model by torchvision name (``pretrained`` is accepted and must be False: no network)."""
    if kw.pop("pretrained", False):
        raise ValueError("pretrained weights are not available offline")
    try:
        return _REGISTRY[name](**kw)
    except KeyError:
        raise ValueError(f"unknown model {name!r}; available: {', '.join(available_models())}") from None


def input_size(model_or_name) -> int:
    """Spatial input size (299 for Inception-v3 — the reference hard-codes 224 and breaks, SURVEY.md Q2; torchvision's
    crop size for EfficientNet-B0 to -B7, 224 to 600, for EfficientNetV2-S / -M / -L, 384 / 480 / 480, and for
    Swin-V2-T / -S / -B, 256; a Vision Transformer's ``image_size``)."""
    if isinstance(model_or_name, str):
        if model_or_name in _EFFICIENTNET_INPUT_SIZE:
            return _EFFICIENTNET_INPUT_SIZE[model_or_name]
        if model_or_name in _EFFICIENTNET_V2_INPUT_SIZE:
            return _EFFICIENTNET_V2_INPUT_SIZE[model_or_name]
        if model_or_name.startswith("swin_v2_"):
            return _SWIN_V2_INPUT_SIZE
        return 299 if model_or_name.startswith("inception") else 224
    return int(getattr(model_or_name, "input_size", 224))
