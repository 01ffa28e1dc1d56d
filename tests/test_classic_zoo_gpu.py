"""GPU tests (H100) of Inception-v3, DenseNet and SqueezeNet: the `classic` group of tools/gpu_diag.py (the channel
concat, max / average / global pooling, stand-alone BN+ReLU and conv+bias+ReLU kernels at every shape these models use
against float64, every Inception-v3 convolution per layer, the models against torchvision with a native-only autograd
graph, and CUDA-graph replay of Inception-v3 and DenseNet-121 training)."""
import os
import subprocess
import sys

import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
pytestmark = pytest.mark.gpu


def test_classic_group():
    r = subprocess.run([sys.executable, os.path.join(ROOT, "tools", "gpu_diag.py"), "--group", "classic"], cwd=ROOT,
                       capture_output=True, text=True, timeout=1500)
    out = r.stdout + r.stderr
    tail = "\n".join(l for l in out.splitlines() if "FAIL" in l or "Error" in l)[:3000] + "\n...\n" + out[-3000:]
    assert r.returncode == 0, tail
    assert "FAIL" not in r.stdout, tail
