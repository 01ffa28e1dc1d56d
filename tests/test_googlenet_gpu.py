"""GPU tests (H100) of GoogLeNet: the `googlenet` group of tools/gpu_diag.py (the segmented BN, adaptive pool and
flatten kernels against float64, the one-node Inception module at all nine module shapes against float64, a native-only
training step, googlenet against torchvision, graph replay), its layer checks under the forced persistent / CTA-pair conv
kernels, the benchmark entry point under graph capture and the ImageNet trainer on googlenet, whose checkpoint loads
into torchvision."""
import json
import os
import subprocess
import sys

import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
pytestmark = pytest.mark.gpu


def _group(name, timeout=1800, env=None):
    e = dict(os.environ)
    e.update(env or {})
    r = subprocess.run([sys.executable, os.path.join(ROOT, "tools", "gpu_diag.py"), "--group", name], cwd=ROOT,
                       capture_output=True, text=True, timeout=timeout, env=e)
    out = r.stdout + r.stderr
    tail = "\n".join(l for l in out.splitlines() if "FAIL" in l or "Error" in l)[:3000] + "\n...\n" + out[-3000:]
    assert r.returncode == 0, tail
    assert "FAIL" not in r.stdout, tail


def test_googlenet_group():
    _group("googlenet")


def test_googlenet_layers_persistent_forced():
    _group("googlenet_layers", env={"DDL_CONV_PERSISTENT": "2", "DDL_CONV_DEEP": "0", "DDL_CONV_AUTOTUNE": "0"})


def test_googlenet_layers_cluster_pairs():
    _group("googlenet_layers", env={"DDL_CONV_CLUSTER": "1", "DDL_CONV_PERSISTENT": "2"})


def _bench(model):
    r = subprocess.run([sys.executable, os.path.join(ROOT, "bench.py"), "--model", model, "--steps", "3", "--warmup", "3"],
                       cwd=ROOT, capture_output=True, text=True, timeout=900)
    assert r.returncode == 0, (r.stdout + r.stderr)[-3000:]
    out = json.loads([l for l in r.stdout.splitlines() if l.startswith("{")][-1])
    for key in ("metric", "value", "unit", "n_gpus", "steps", "warmup", "ms_per_step", "higher_is_better", "scaling",
                "vs_baseline", "dtype", "data", "config", "clocks", "e2e", "gpu_launches"):
        assert key in out, key
    assert out["value"] > 0 and out["gpu_launches"] > 0 and out["e2e"]["value"] > 0
    assert out["config"]["cuda_graph"] is True and out["config"]["model"] == model


def test_bench_googlenet():
    _bench("googlenet")


def test_imagenet_trainer_googlenet(tmp_path):
    sys.path.insert(0, ROOT)
    import io

    import torch
    import torchvision

    from distributeddeeplearning_b200.cli import launcher

    out, err = io.StringIO(), io.StringIO()
    res = launcher.launch("distributeddeeplearning_b200.workloads.imagenet",
                          ["--epochs", "1", "--batch_size", "16", "--model", "googlenet",
                           "--save_filepath", str(tmp_path / "ck-{epoch}.pt")], gpus=1, record=False, stdout=out,
                          stderr=err, timeout=900, env={"PYTHONPATH": ROOT, "FAKE_DATA_LENGTH": "64"})
    assert res.returncode == 0, (out.getvalue() + err.getvalue())[-3000:]
    assert "Training epoch 0 took" in out.getvalue()
    state = torch.load(tmp_path / "ck-1.pt", map_location="cpu", weights_only=False)
    torchvision.models.googlenet(init_weights=True).load_state_dict(state["model"], strict=True)
