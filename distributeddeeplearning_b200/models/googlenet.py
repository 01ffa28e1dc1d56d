"""GoogLeNet (keys, shapes and initialisation match ``torchvision.models.googlenet``).

Each Inception module runs as one autograd node, ``ops.inception_module``: the three 1x1 convolutions that read the
module input are one GEMM, and the branch BatchNorms write their slices of the output in place (ops/googlenet.py).
The stem layers are ``conv_bn`` units; the pools use ``ceil_mode=True``, as torchvision's do.  torchvision's known
quirk is kept: the "5x5" branch uses a 3x3 kernel.

The auxiliary heads (training only) pool 14x14 maps to 4x4 with torch's adaptive windows, run a 1x1 ``BasicConv2d`` to
128 channels, flatten in torchvision's NCHW order and apply fc1 + ReLU, dropout and fc2, all natively on CUDA.  In
training with aux heads the model returns ``GoogLeNetOutputs(logits, aux_logits2, aux_logits1)``, torchvision's order;
``aux_loss_weight`` is the weight of each auxiliary loss (0.3, the paper's discount weight).
"""
from __future__ import annotations

from collections import namedtuple

import torch
import torch.nn as nn

from .. import ops
from .inception import BasicConv2d
from .layers import BatchNorm2d, Conv2d, Linear, conv_bn, prepare_input

GoogLeNetOutputs = namedtuple("GoogLeNetOutputs", ["logits", "aux_logits2", "aux_logits1"])


class Inception(nn.Module):
    def __init__(self, cin, ch1x1, ch3x3red, ch3x3, ch5x5red, ch5x5, pool_proj):
        super().__init__()
        self.branch1 = BasicConv2d(cin, ch1x1, 1)
        self.branch2 = nn.Sequential(BasicConv2d(cin, ch3x3red, 1), BasicConv2d(ch3x3red, ch3x3, 3, padding=1))
        self.branch3 = nn.Sequential(BasicConv2d(cin, ch5x5red, 1), BasicConv2d(ch5x5red, ch5x5, 3, padding=1))
        # index 0 holds no parameters (the pool runs inside the node), so branch4.1 keeps torchvision's keys
        self.branch4 = nn.Sequential(nn.MaxPool2d(3, 1, 1, ceil_mode=True), BasicConv2d(cin, pool_proj, 1))

    def forward(self, x):
        return ops.inception_module(x, (self.branch1, self.branch2[0], self.branch2[1], self.branch3[0],
                                        self.branch3[1], self.branch4[1]))


class InceptionAux(nn.Module):
    def __init__(self, cin, num_classes, dropout=0.7):
        super().__init__()
        self.conv = BasicConv2d(cin, 128, 1)
        self.fc1 = Linear(2048, 1024)
        self.fc2 = Linear(1024, num_classes)
        self.p, self.num_classes = dropout, num_classes

    def forward(self, x):
        x = ops.adaptive_avg_pool2d(x, (4, 4))
        x = ops.flatten_nchw(self.conv(x))
        x = ops.dropout(self.fc1(x, relu=True), self.p, self.training)
        return self.fc2(x)[:, : self.num_classes]


class GoogLeNet(nn.Module):
    input_size = 224
    aux_loss_weight = 0.3

    def __init__(self, num_classes=1000, aux_logits=True, transform_input=False, init_weights=None, blocks=None,
                 dropout=0.2, dropout_aux=0.7):
        super().__init__()
        if blocks is not None:
            raise ValueError("GoogLeNet: custom blocks are not supported; the modules run on the native Inception node")
        self.num_classes, self.aux_logits, self.transform_input, self.p = num_classes, aux_logits, transform_input, dropout
        self.conv1 = BasicConv2d(3, 64, 7, stride=2, padding=3)
        self.maxpool1 = nn.MaxPool2d(3, stride=2, ceil_mode=True)
        self.conv2 = BasicConv2d(64, 64, 1)
        self.conv3 = BasicConv2d(64, 192, 3, padding=1)
        self.maxpool2 = nn.MaxPool2d(3, stride=2, ceil_mode=True)
        self.inception3a = Inception(192, 64, 96, 128, 16, 32, 32)
        self.inception3b = Inception(256, 128, 128, 192, 32, 96, 64)
        self.maxpool3 = nn.MaxPool2d(3, stride=2, ceil_mode=True)
        self.inception4a = Inception(480, 192, 96, 208, 16, 48, 64)
        self.inception4b = Inception(512, 160, 112, 224, 24, 64, 64)
        self.inception4c = Inception(512, 128, 128, 256, 24, 64, 64)
        self.inception4d = Inception(512, 112, 144, 288, 32, 64, 64)
        self.inception4e = Inception(528, 256, 160, 320, 32, 128, 128)
        self.maxpool4 = nn.MaxPool2d(2, stride=2, ceil_mode=True)
        self.inception5a = Inception(832, 256, 160, 320, 32, 128, 128)
        self.inception5b = Inception(832, 384, 192, 384, 48, 128, 128)
        if aux_logits:
            self.aux1 = InceptionAux(512, num_classes, dropout=dropout_aux)
            self.aux2 = InceptionAux(528, num_classes, dropout=dropout_aux)
        else:
            self.aux1 = self.aux2 = None
        self.fc = Linear(1024, num_classes)
        if init_weights is None or init_weights:
            for m in self.modules():
                if isinstance(m, (Conv2d, Linear)):
                    nn.init.trunc_normal_(m.weight, mean=0.0, std=0.01, a=-2, b=2)
                elif isinstance(m, BatchNorm2d):
                    nn.init.constant_(m.weight, 1)
                    nn.init.constant_(m.bias, 0)

    def _transform_input(self, x):
        """torchvision's per-channel affine of the three image channels (ImageNet statistics -> the (0.5, 0.5)
        normalisation the original weights expect); the zero pad channel of an NHWC4 image stays zero."""
        dt = torch.float32 if x.dtype in (torch.bfloat16, torch.float16) else x.dtype
        scale = torch.tensor([0.229 / 0.5, 0.224 / 0.5, 0.225 / 0.5], dtype=dt, device=x.device)
        shift = torch.tensor([(0.485 - 0.5) / 0.5, (0.456 - 0.5) / 0.5, (0.406 - 0.5) / 0.5], dtype=dt, device=x.device)
        if x.shape[1] == 4:
            scale, shift = torch.cat([scale, scale.new_zeros(1)]), torch.cat([shift, shift.new_zeros(1)])
        y = x.to(dt) * scale.view(1, -1, 1, 1) + shift.view(1, -1, 1, 1)
        return y.to(x.dtype).contiguous(memory_format=torch.channels_last) if x.is_cuda else y.to(x.dtype)

    def forward(self, x):
        if self.transform_input:
            x = self._transform_input(x)
        x = prepare_input(x)
        x = self.conv1(x)
        x = ops.max_pool2d(x, 3, 2, ceil_mode=True)
        x = self.conv3(self.conv2(x))
        x = ops.max_pool2d(x, 3, 2, ceil_mode=True)
        x = self.inception3b(self.inception3a(x))
        x = ops.max_pool2d(x, 3, 2, ceil_mode=True)
        x = self.inception4a(x)
        aux = self.training and self.aux_logits
        aux1 = self.aux1(x) if aux else None
        x = self.inception4d(self.inception4c(self.inception4b(x)))
        aux2 = self.aux2(x) if aux else None
        x = self.inception4e(x)
        x = ops.max_pool2d(x, 2, 2, ceil_mode=True)
        x = self.inception5b(self.inception5a(x))
        x = ops.global_avg_pool(x)
        x = ops.dropout(x, self.p, self.training)
        x = self.fc(x)[:, : self.num_classes]
        return GoogLeNetOutputs(x, aux2, aux1) if aux else x


def googlenet(**kw):
    return GoogLeNet(**kw)
