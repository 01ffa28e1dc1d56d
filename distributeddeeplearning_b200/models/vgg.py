"""VGG-11/13/16/19 (+BN variants) — the large-gradient allreduce stress model (527.8 MiB fp32 for
VGG-16, one 392 MiB FC tensor; SURVEY.md 2.7).  Keys match ``torchvision.models.vgg*``.

conv+bias+ReLU is one wgmma kernel (bias/ReLU in the epilogue, SURVEY.md K20); the three FC
layers are the same GEMM kernel; dropout recomputes its Philox mask in backward.
"""
from __future__ import annotations

import torch.nn as nn

from .. import ops
from .layers import BatchNorm2d, Conv2d, Linear, conv_bn, prepare_input

cfgs = {
    "A": [64, "M", 128, "M", 256, 256, "M", 512, 512, "M", 512, 512, "M"],
    "B": [64, 64, "M", 128, 128, "M", 256, 256, "M", 512, 512, "M", 512, 512, "M"],
    "D": [64, 64, "M", 128, 128, "M", 256, 256, 256, "M", 512, 512, 512, "M", 512, 512, 512, "M"],
    "E": [64, 64, "M", 128, 128, "M", 256, 256, 256, 256, "M", 512, 512, 512, 512, "M", 512, 512, 512, 512, "M"],
}


class _Pool(nn.Module):
    def forward(self, x):
        return ops.max_pool2d(x, 2, 2, 0)


class _ReLUMarker(nn.Module):
    """Placeholder keeping torchvision's Sequential indices (ReLU is fused into the conv)."""

    def forward(self, x):
        return x


class VGG(nn.Module):
    input_size = 224

    def __init__(self, cfg, batch_norm=False, num_classes=1000, dropout=0.5):
        super().__init__()
        self.num_classes, self.p = num_classes, dropout
        layers, cin = [], 3
        for v in cfg:
            if v == "M":
                layers.append(_Pool())
            else:
                layers.append(Conv2d(cin, v, 3, 1, 1, bias=True))
                if batch_norm:
                    layers.append(BatchNorm2d(v))
                layers.append(_ReLUMarker())
                cin = v
        self.features = nn.Sequential(*layers)
        self.batch_norm = batch_norm
        self.classifier = nn.Sequential(Linear(512 * 7 * 7, 4096), _ReLUMarker(), _ReLUMarker(), Linear(4096, 4096),
                                        _ReLUMarker(), _ReLUMarker(), Linear(4096, num_classes))
        for m in self.modules():
            if isinstance(m, Conv2d):
                nn.init.kaiming_normal_(m.weight, mode="fan_out", nonlinearity="relu")
                if m.bias is not None:
                    nn.init.zeros_(m.bias)
            elif isinstance(m, Linear):
                nn.init.normal_(m.weight, 0, 0.01)
                nn.init.zeros_(m.bias)

    def forward(self, x):
        x = prepare_input(x)
        mods = list(self.features)
        i = 0
        while i < len(mods):
            m = mods[i]
            if isinstance(m, Conv2d):
                if self.batch_norm:
                    # train-mode BN subtracts the batch mean, so the conv bias cancels exactly (its
                    # gradient is identically zero); the parameter is kept for state_dict parity only
                    x = conv_bn(x, m, mods[i + 1], relu=True)
                    i += 3
                else:
                    x = m(x, relu=True)
                    i += 2
            else:
                x = m(x)
                i += 1
        # torchvision flattens in logical (c, h, w) order; reshape() of the channels_last tensor does
        # exactly that (one 12.8 MB copy at batch 256), keeping FC weights checkpoint-compatible
        x = x.reshape(x.shape[0], -1)
        x = self.classifier[0](x, relu=True)
        x = ops.dropout(x, self.p, self.training)
        x = self.classifier[3](x, relu=True)
        x = ops.dropout(x, self.p, self.training)
        return self.classifier[6](x)[:, : self.num_classes]


def _vgg(cfg, bn, **kw):
    return VGG(cfgs[cfg], batch_norm=bn, **kw)


def vgg11(**kw): return _vgg("A", False, **kw)
def vgg13(**kw): return _vgg("B", False, **kw)
def vgg16(**kw): return _vgg("D", False, **kw)
def vgg19(**kw): return _vgg("E", False, **kw)
def vgg11_bn(**kw): return _vgg("A", True, **kw)
def vgg13_bn(**kw): return _vgg("B", True, **kw)
def vgg16_bn(**kw): return _vgg("D", True, **kw)
def vgg19_bn(**kw): return _vgg("E", True, **kw)
