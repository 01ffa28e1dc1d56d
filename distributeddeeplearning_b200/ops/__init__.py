"""Fused ops: hand-written sm_90a kernels on CUDA, PyTorch composites on CPU (see functional.py)."""
from .convnext import convnext_block, layer_norm_channels  # noqa: F401
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
    hardswish,
    linear,
    max_pool2d,
    seed_dropout,
    softmax_cross_entropy,
    squeeze_excite,
    stochastic_depth_keep,
    topk_correct,
    use_native,
)
from .maxvit import grid_attention, maxvit_attention_layer  # noqa: F401
from .swin import patch_merging, swin_block, window_attention  # noqa: F401
from .swin_v2 import patch_merging_v2, swin_v2_block, window_attention_v2  # noqa: F401
from .vit import self_attention, vit_embed, vit_encoder_block  # noqa: F401
