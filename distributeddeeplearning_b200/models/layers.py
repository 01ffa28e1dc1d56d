"""Parameter containers + fused layer helpers shared by the model zoo.

Modules keep torchvision's attribute names (``conv1``, ``bn1``, ``layer1.0.conv2`` ...) so
``state_dict`` keys match ``torchvision.models`` one-for-one (the reference builds its models
with ``getattr(torchvision.models, name)()`` — ``pytorch_synthetic_benchmark.py:60``) and
checkpoints are interchangeable.  Compute does not go through ``nn.Conv2d.forward`` /
``nn.BatchNorm2d.forward``: blocks call the fused ops in ``ops.functional`` with these
containers' tensors.  Conv weights are stored ``channels_last`` (KRSC) so the fp32 master,
its bf16 GEMM copy and the wgrad output share one flat layout.
"""
from __future__ import annotations

import math

import torch
import torch.nn as nn

from .. import ops

CL = torch.channels_last


class Conv2d(nn.Module):
    """Weight (and optional bias) holder for a convolution."""

    def __init__(self, cin, cout, kernel_size, stride=1, padding=0, dilation=1, bias=False, groups=1):
        super().__init__()
        ks = (kernel_size, kernel_size) if isinstance(kernel_size, int) else tuple(kernel_size)
        if cin % groups != 0 or cout % groups != 0:
            raise ValueError("in_channels and out_channels must be divisible by groups")
        self.in_channels, self.out_channels = cin, cout
        self.kernel_size, self.stride, self.padding, self.dilation = ks, stride, padding, dilation
        self.groups = groups
        w = torch.empty(cout, cin // groups, *ks).contiguous(memory_format=CL)
        self.weight = nn.Parameter(w)
        self.weight._ddl_groups = groups     # a grouped [Cout, Cin/groups, R, S] weight is never a stem weight
        self.bias = nn.Parameter(torch.zeros(cout)) if bias else None
        self.reset_parameters()

    def reset_parameters(self):
        nn.init.kaiming_uniform_(self.weight, a=math.sqrt(5))
        if self.bias is not None:
            fan_in = self.weight.shape[1] * self.kernel_size[0] * self.kernel_size[1]
            bound = 1 / math.sqrt(fan_in)
            nn.init.uniform_(self.bias, -bound, bound)

    def _load_from_state_dict(self, state_dict, prefix, *a, **k):
        key = prefix + "weight"
        if key in state_dict:
            state_dict[key] = state_dict[key].contiguous(memory_format=CL)
        super()._load_from_state_dict(state_dict, prefix, *a, **k)

    def forward(self, x, relu=False):
        """Standalone conv (+bias, +ReLU) — VGG / AlexNet style layers."""
        return ops.conv_bias_act(x, self.weight, self.bias, self.stride, self.padding, self.dilation, relu, self.groups)

    def extra_repr(self):
        return f"{self.in_channels}, {self.out_channels}, kernel_size={self.kernel_size}, stride={self.stride}, padding={self.padding}" + \
            (f", groups={self.groups}" if self.groups != 1 else "")


class BatchNorm2d(nn.Module):
    """Affine parameters + running statistics holder (same state_dict as nn.BatchNorm2d)."""

    def __init__(self, num_features, eps=1e-5, momentum=0.1):
        super().__init__()
        self.num_features, self.eps, self.momentum = num_features, eps, momentum
        self.weight = nn.Parameter(torch.ones(num_features))
        self.bias = nn.Parameter(torch.zeros(num_features))
        self.register_buffer("running_mean", torch.zeros(num_features))
        self.register_buffer("running_var", torch.ones(num_features))
        self.register_buffer("num_batches_tracked", torch.tensor(0, dtype=torch.long))

    def extra_repr(self):
        return f"{self.num_features}, eps={self.eps}, momentum={self.momentum}"


class LayerNorm(nn.Module):
    """Affine parameters holder of a LayerNorm over channels (same state_dict as nn.LayerNorm(C)); ``forward``
    normalises the channels of an NHWC activation [N, C, H, W] or of a matrix [N, C]."""

    def __init__(self, num_features, eps=1e-5):
        super().__init__()
        self.normalized_shape, self.eps = (num_features,), eps
        self.weight = nn.Parameter(torch.ones(num_features))
        self.bias = nn.Parameter(torch.zeros(num_features))

    def forward(self, x):
        return ops.layer_norm_channels(x, self.weight, self.bias, self.eps)

    def extra_repr(self):
        return f"{self.normalized_shape}, eps={self.eps}"


def conv_bn(x, conv: Conv2d, bn: BatchNorm2d, relu=True, residual=None, relu6=False, hardswish=False, silu=False,
            sample_scale=None):
    """act(BN(conv(x)) [+ residual]) through the fused op (``relu6``: the activation is ReLU6; ``hardswish``: it is
    hardswish; ``silu``: it is SiLU).  ``sample_scale``: per-sample scales of stochastic depth applied to the BN output
    before the residual add (no activation)."""
    return ops.conv_bn_act(x, conv.weight, bn.weight, bn.bias, bn.running_mean, bn.running_var, conv.stride,
                           conv.padding,
                           conv.dilation, bn.eps, bn.momentum, relu, residual, bn.training,
                           **({"groups": conv.groups} if conv.groups != 1 else {}),
                           **({"relu6": True} if relu6 else {}),
                           **({"hardswish": True} if hardswish else {}),
                           **({"silu": True} if silu else {}),
                           **({"sample_scale": sample_scale} if sample_scale is not None else {}))


def conv_bn_pool(x, conv: Conv2d, bn: BatchNorm2d, kernel=3, stride=2, padding=1):
    """maxpool(relu(BN(conv(x)))) — stem unit (fused on the native training path)."""
    return ops.conv_bn_act_maxpool(x, conv.weight, bn.weight, bn.bias, bn.running_mean, bn.running_var, conv.stride,
                                   conv.padding, conv.dilation, bn.eps, bn.momentum, bn.training, kernel, stride, padding)


def bn_act(x, bn: BatchNorm2d, relu=True):
    """act(BN(x)) on its own (pre-activation networks)."""
    return ops.batch_norm_act(x, bn.weight, bn.bias, bn.running_mean, bn.running_var, bn.eps, bn.momentum, relu,
                              bn.training)


class Linear(nn.Module):
    def __init__(self, in_features, out_features, bias=True):
        super().__init__()
        self.in_features, self.out_features = in_features, out_features
        self.weight = nn.Parameter(torch.empty(out_features, in_features))
        self.bias = nn.Parameter(torch.zeros(out_features)) if bias else None
        nn.init.kaiming_uniform_(self.weight, a=math.sqrt(5))
        if bias:
            bound = 1 / math.sqrt(in_features)
            nn.init.uniform_(self.bias, -bound, bound)

    def forward(self, x, relu=False):
        return ops.linear(x, self.weight, self.bias, relu)

    def extra_repr(self):
        return f"in_features={self.in_features}, out_features={self.out_features}"


def prepare_input(x: torch.Tensor) -> torch.Tensor:
    """Bring an image batch into the layout/dtype the active device path expects.

    CUDA: bf16 NHWC4 (logical [N,4,H,W] channels_last, zero 4th channel).  CPU: unchanged fp32.
    """
    if not x.is_cuda or not ops.use_native(x):
        if x.is_cuda and x.dtype != torch.bfloat16:
            x = x.to(torch.bfloat16)
        return x.contiguous(memory_format=CL) if x.is_cuda else x
    if x.dtype == torch.bfloat16 and x.shape[1] == 4 and x.is_contiguous(memory_format=CL):
        return x
    from ..ops import native

    if x.shape[1] > 4:
        raise ValueError("image input must have <= 4 channels")
    return native.nchw_to_nhwc4(x)
