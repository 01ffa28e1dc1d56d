"""GPU tests (H100) of the depthwise kernels, ReLU6 BatchNorm and MobileNetV2: the `depthwise` and `mobilenet` groups of
tools/gpu_diag.py (one subprocess each, as in test_gpu.py), the benchmark entry point and the ImageNet trainer on
mobilenet_v2."""
import json
import os
import subprocess
import sys

import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
pytestmark = pytest.mark.gpu


def _group(name, timeout=900, env=None):
    e = dict(os.environ)
    e.update(env or {})
    r = subprocess.run([sys.executable, os.path.join(ROOT, "tools", "gpu_diag.py"), "--group", name], cwd=ROOT,
                       capture_output=True, text=True, timeout=timeout, env=e)
    out = r.stdout + r.stderr
    tail = "\n".join(l for l in out.splitlines() if "FAIL" in l or "Error" in l)[:3000] + "\n...\n" + out[-3000:]
    assert r.returncode == 0, tail
    assert "FAIL" not in r.stdout, tail


def test_depthwise_group():
    """Depthwise fwd / dgrad / wgrad per shape, ReLU6 BN in both mask modes, inverted-residual blocks vs float64."""
    _group("depthwise")


def test_mobilenet_group():
    """mobilenet_v2 vs torchvision (train gradients, eval logits), eager vs graph replay, fp8 session."""
    _group("mobilenet")


def test_bench_mobilenet_v2():
    r = subprocess.run([sys.executable, os.path.join(ROOT, "bench.py"), "--model", "mobilenet_v2", "--steps", "3",
                        "--warmup", "3", "--batch-size", "32"], cwd=ROOT, capture_output=True, text=True, timeout=900)
    assert r.returncode == 0, (r.stdout + r.stderr)[-3000:]
    out = json.loads([l for l in r.stdout.splitlines() if l.startswith("{")][-1])
    for key in ("metric", "value", "unit", "n_gpus", "steps", "warmup", "ms_per_step", "higher_is_better", "scaling",
                "vs_baseline", "dtype", "data", "config", "clocks", "e2e", "gpu_launches"):
        assert key in out, key
    assert out["value"] > 0 and out["gpu_launches"] > 0 and out["e2e"]["value"] > 0
    assert out["config"]["model"] == "mobilenet_v2" and out["config"]["cuda_graph"] is True


def test_imagenet_trainer_mobilenet_v2(tmp_path):
    sys.path.insert(0, ROOT)
    import io

    from distributeddeeplearning_b200.cli import launcher

    out, err = io.StringIO(), io.StringIO()
    res = launcher.launch("distributeddeeplearning_b200.workloads.imagenet",
                          ["--epochs", "1", "--batch_size", "16", "--model", "mobilenet_v2",
                           "--save_filepath", str(tmp_path / "ck-{epoch}.pt")], gpus=1, record=False, stdout=out,
                          stderr=err, timeout=900, env={"PYTHONPATH": ROOT, "FAKE_DATA_LENGTH": "64"})
    assert res.returncode == 0, (out.getvalue() + err.getvalue())[-3000:]
    assert "Training epoch 0 took" in out.getvalue()
