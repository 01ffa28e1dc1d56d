"""ddl: an H100-native distributed-training benchmark harness.

Capabilities of microsoft/DistributedDeepLearning's PyTorch templates
(PyTorch_benchmark / PyTorch_imagenet / PyTorch_hvd; the TensorFlow twins
collapse onto them), rebuilt for one 8xH100 NVSwitch box:

* ``cli``        local launcher + task tree (replaces cookiecutter/AzureML control plane)
* ``workloads``  synthetic benchmark, ImageNet trainer, resume-capable trainer
* ``parallel``   Horovod-equivalent API, static bucket plan, fused allreduce+SGD over
                 NVLink peer / NVLS multicast memory
* ``ops``        hand-written sm_90a kernels (wgmma/TMA conv-GEMMs, fused BN,
                 softmax-xent, pools, Philox synthetic data) + fp32 PyTorch references
* ``models``     ResNet-50/101/152 (+18/34), VGG, AlexNet, Inception-v3
* ``data``       synthetic datasets, ImageFolder pipeline, samplers, ImageNet prep
* ``utils``      timers, meters, LR schedule, checkpoint/resume, run history, config
"""

__version__ = "0.1.0"

from . import utils  # noqa: F401
