"""Inception-v3 with auxiliary classifier (299x299 input).

Keys match ``torchvision.models.inception_v3``.  The reference cannot actually run this model
(``--model inception_v3`` feeds 224x224 and passes the (logits, aux) tuple to ``cross_entropy`` —
SURVEY.md Q2); here the workloads size the input from ``model.input_size`` and add the 0.4-weighted
auxiliary loss.

Every layer runs on the wgmma conv kernels: Inception's widths (32/48/80/96/192/288/320/448 ...) are multiples
of 8, which is all the kernels need (partial 64-channel k-blocks are zero-filled by TMA, partial N tiles masked), and
the 1x7 / 7x1 kernels use per-axis padding.  Branch outputs are concatenated by ``ops.concat_channels`` (one native
gather kernel forward, one scatter kernel backward).
"""
from __future__ import annotations

import torch.nn as nn

from .. import ops
from .layers import BatchNorm2d, Conv2d, Linear, conv_bn, prepare_input


class BasicConv2d(nn.Module):
    def __init__(self, cin, cout, kernel_size, stride=1, padding=0):
        super().__init__()
        self.conv = Conv2d(cin, cout, kernel_size, stride, padding)
        self.bn = BatchNorm2d(cout, eps=0.001)

    def forward(self, x):
        return conv_bn(x, self.conv, self.bn, relu=True)


def _cat(xs):
    return ops.concat_channels(xs)


class InceptionA(nn.Module):
    def __init__(self, cin, pool_features):
        super().__init__()
        self.branch1x1 = BasicConv2d(cin, 64, 1)
        self.branch5x5_1 = BasicConv2d(cin, 48, 1)
        self.branch5x5_2 = BasicConv2d(48, 64, 5, padding=2)
        self.branch3x3dbl_1 = BasicConv2d(cin, 64, 1)
        self.branch3x3dbl_2 = BasicConv2d(64, 96, 3, padding=1)
        self.branch3x3dbl_3 = BasicConv2d(96, 96, 3, padding=1)
        self.branch_pool = BasicConv2d(cin, pool_features, 1)

    def forward(self, x):
        b1 = self.branch1x1(x)
        b5 = self.branch5x5_2(self.branch5x5_1(x))
        b3 = self.branch3x3dbl_3(self.branch3x3dbl_2(self.branch3x3dbl_1(x)))
        bp = self.branch_pool(ops.avg_pool2d(x, 3, 1, 1))
        return _cat([b1, b5, b3, bp])


class InceptionB(nn.Module):
    def __init__(self, cin):
        super().__init__()
        self.branch3x3 = BasicConv2d(cin, 384, 3, stride=2)
        self.branch3x3dbl_1 = BasicConv2d(cin, 64, 1)
        self.branch3x3dbl_2 = BasicConv2d(64, 96, 3, padding=1)
        self.branch3x3dbl_3 = BasicConv2d(96, 96, 3, stride=2)

    def forward(self, x):
        b3 = self.branch3x3(x)
        bd = self.branch3x3dbl_3(self.branch3x3dbl_2(self.branch3x3dbl_1(x)))
        bp = ops.max_pool2d(x, 3, 2)
        return _cat([b3, bd, bp])


class InceptionC(nn.Module):
    def __init__(self, cin, c7):
        super().__init__()
        self.branch1x1 = BasicConv2d(cin, 192, 1)
        self.branch7x7_1 = BasicConv2d(cin, c7, 1)
        self.branch7x7_2 = BasicConv2d(c7, c7, (1, 7), padding=(0, 3))
        self.branch7x7_3 = BasicConv2d(c7, 192, (7, 1), padding=(3, 0))
        self.branch7x7dbl_1 = BasicConv2d(cin, c7, 1)
        self.branch7x7dbl_2 = BasicConv2d(c7, c7, (7, 1), padding=(3, 0))
        self.branch7x7dbl_3 = BasicConv2d(c7, c7, (1, 7), padding=(0, 3))
        self.branch7x7dbl_4 = BasicConv2d(c7, c7, (7, 1), padding=(3, 0))
        self.branch7x7dbl_5 = BasicConv2d(c7, 192, (1, 7), padding=(0, 3))
        self.branch_pool = BasicConv2d(cin, 192, 1)

    def forward(self, x):
        b1 = self.branch1x1(x)
        b7 = self.branch7x7_3(self.branch7x7_2(self.branch7x7_1(x)))
        bd = self.branch7x7dbl_1(x)
        for m in (self.branch7x7dbl_2, self.branch7x7dbl_3, self.branch7x7dbl_4, self.branch7x7dbl_5):
            bd = m(bd)
        bp = self.branch_pool(ops.avg_pool2d(x, 3, 1, 1))
        return _cat([b1, b7, bd, bp])


class InceptionD(nn.Module):
    def __init__(self, cin):
        super().__init__()
        self.branch3x3_1 = BasicConv2d(cin, 192, 1)
        self.branch3x3_2 = BasicConv2d(192, 320, 3, stride=2)
        self.branch7x7x3_1 = BasicConv2d(cin, 192, 1)
        self.branch7x7x3_2 = BasicConv2d(192, 192, (1, 7), padding=(0, 3))
        self.branch7x7x3_3 = BasicConv2d(192, 192, (7, 1), padding=(3, 0))
        self.branch7x7x3_4 = BasicConv2d(192, 192, 3, stride=2)

    def forward(self, x):
        b3 = self.branch3x3_2(self.branch3x3_1(x))
        b7 = self.branch7x7x3_4(self.branch7x7x3_3(self.branch7x7x3_2(self.branch7x7x3_1(x))))
        bp = ops.max_pool2d(x, 3, 2)
        return _cat([b3, b7, bp])


class InceptionE(nn.Module):
    def __init__(self, cin):
        super().__init__()
        self.branch1x1 = BasicConv2d(cin, 320, 1)
        self.branch3x3_1 = BasicConv2d(cin, 384, 1)
        self.branch3x3_2a = BasicConv2d(384, 384, (1, 3), padding=(0, 1))
        self.branch3x3_2b = BasicConv2d(384, 384, (3, 1), padding=(1, 0))
        self.branch3x3dbl_1 = BasicConv2d(cin, 448, 1)
        self.branch3x3dbl_2 = BasicConv2d(448, 384, 3, padding=1)
        self.branch3x3dbl_3a = BasicConv2d(384, 384, (1, 3), padding=(0, 1))
        self.branch3x3dbl_3b = BasicConv2d(384, 384, (3, 1), padding=(1, 0))
        self.branch_pool = BasicConv2d(cin, 192, 1)

    def forward(self, x):
        b1 = self.branch1x1(x)
        b3 = self.branch3x3_1(x)
        b3 = _cat([self.branch3x3_2a(b3), self.branch3x3_2b(b3)])
        bd = self.branch3x3dbl_2(self.branch3x3dbl_1(x))
        bd = _cat([self.branch3x3dbl_3a(bd), self.branch3x3dbl_3b(bd)])
        bp = self.branch_pool(ops.avg_pool2d(x, 3, 1, 1))
        return _cat([b1, b3, bd, bp])


class InceptionAux(nn.Module):
    def __init__(self, cin, num_classes):
        super().__init__()
        self.conv0 = BasicConv2d(cin, 128, 1)
        self.conv1 = BasicConv2d(128, 768, 5)
        self.fc = Linear(768, num_classes)
        self.num_classes = num_classes

    def forward(self, x):
        x = ops.avg_pool2d(x, 5, 3)
        x = self.conv1(self.conv0(x))
        x = ops.global_avg_pool(x)
        return self.fc(x)[:, : self.num_classes]


class Inception3(nn.Module):
    input_size = 299
    aux_loss_weight = 0.4          # the auxiliary head's weight in the training loss (ops.aux_classification_loss)

    def __init__(self, num_classes=1000, aux_logits=True, dropout=0.5):
        super().__init__()
        self.num_classes, self.aux_logits, self.p = num_classes, aux_logits, dropout
        self.Conv2d_1a_3x3 = BasicConv2d(3, 32, 3, stride=2)
        self.Conv2d_2a_3x3 = BasicConv2d(32, 32, 3)
        self.Conv2d_2b_3x3 = BasicConv2d(32, 64, 3, padding=1)
        self.Conv2d_3b_1x1 = BasicConv2d(64, 80, 1)
        self.Conv2d_4a_3x3 = BasicConv2d(80, 192, 3)
        self.Mixed_5b = InceptionA(192, 32)
        self.Mixed_5c = InceptionA(256, 64)
        self.Mixed_5d = InceptionA(288, 64)
        self.Mixed_6a = InceptionB(288)
        self.Mixed_6b = InceptionC(768, 128)
        self.Mixed_6c = InceptionC(768, 160)
        self.Mixed_6d = InceptionC(768, 160)
        self.Mixed_6e = InceptionC(768, 192)
        self.AuxLogits = InceptionAux(768, num_classes) if aux_logits else None
        self.Mixed_7a = InceptionD(768)
        self.Mixed_7b = InceptionE(1280)
        self.Mixed_7c = InceptionE(2048)
        self.fc = Linear(2048, num_classes)
        for m in self.modules():
            if isinstance(m, (Conv2d, Linear)):
                nn.init.trunc_normal_(m.weight, mean=0.0, std=0.1, a=-2, b=2)

    def forward(self, x):
        x = prepare_input(x)
        x = self.Conv2d_2b_3x3(self.Conv2d_2a_3x3(self.Conv2d_1a_3x3(x)))
        x = ops.max_pool2d(x, 3, 2)
        x = self.Conv2d_4a_3x3(self.Conv2d_3b_1x1(x))
        x = ops.max_pool2d(x, 3, 2)
        x = self.Mixed_5d(self.Mixed_5c(self.Mixed_5b(x)))
        x = self.Mixed_6a(x)
        x = self.Mixed_6e(self.Mixed_6d(self.Mixed_6c(self.Mixed_6b(x))))
        aux = self.AuxLogits(x) if (self.training and self.AuxLogits is not None) else None
        x = self.Mixed_7c(self.Mixed_7b(self.Mixed_7a(x)))
        x = ops.global_avg_pool(x)
        x = ops.dropout(x, self.p, self.training)
        out = self.fc(x)[:, : self.num_classes]
        return (out, aux) if aux is not None else out


def inception_v3(**kw):
    return Inception3(**kw)
