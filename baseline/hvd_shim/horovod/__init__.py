"""Compatibility shim: `import horovod.torch as hvd` on top of torch.distributed (NCCL / gloo).

Only used by the REFERENCE ARM of bench.py to run the reference's unmodified
pytorch_synthetic_benchmark.py on a box where horovod==0.15.2 / torch==1.0.0 / CUDA 9 cannot be
installed (no sm_90 support, no wheels offline).  None of b200-ddl's models, kernels or engine are
on this path: it is stock torchvision + cuDNN + NCCL, i.e. what the reference would execute today.
"""
