"""Fused ops: hand-written sm_90a kernels on CUDA, PyTorch composites on CPU (see functional.py)."""
from .functional import (  # noqa: F401
    advance_dropout_step,
    avg_pool2d,
    batch_norm_act,
    concat_channels,
    conv_bias_act,
    conv_bn_act,
    conv_bn_act_maxpool,
    dropout,
    global_avg_pool,
    linear,
    max_pool2d,
    seed_dropout,
    softmax_cross_entropy,
    topk_correct,
    use_native,
)
