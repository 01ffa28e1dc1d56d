"""GPU tests (H100) of the Vision Transformer: the `vit` group of tools/gpu_diag.py (attention forward and backward at
every zoo shape and edge cases, add + LayerNorm, LayerNorm backward with an addend, patchify, token assembly, vit_b_16
against torchvision, graph replay and an fp8 session), the benchmark entry point and the ImageNet trainer on vit_b_32."""
import json
import os
import subprocess
import sys

import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
pytestmark = pytest.mark.gpu


def test_vit_group():
    r = subprocess.run([sys.executable, os.path.join(ROOT, "tools", "gpu_diag.py"), "--group", "vit"], cwd=ROOT,
                       capture_output=True, text=True, timeout=1500)
    out = r.stdout + r.stderr
    tail = "\n".join(l for l in out.splitlines() if "FAIL" in l or "Error" in l)[:3000] + "\n...\n" + out[-3000:]
    assert r.returncode == 0, tail
    assert "FAIL" not in r.stdout, tail


def test_bench_vit_b_16():
    r = subprocess.run([sys.executable, os.path.join(ROOT, "bench.py"), "--model", "vit_b_16", "--steps", "3",
                        "--warmup", "3", "--batch-size", "32"], cwd=ROOT, capture_output=True, text=True, timeout=900)
    assert r.returncode == 0, (r.stdout + r.stderr)[-3000:]
    out = json.loads([l for l in r.stdout.splitlines() if l.startswith("{")][-1])
    for key in ("metric", "value", "unit", "n_gpus", "steps", "warmup", "ms_per_step", "higher_is_better", "scaling",
                "vs_baseline", "dtype", "data", "config", "clocks", "e2e", "gpu_launches"):
        assert key in out, key
    assert out["value"] > 0 and out["gpu_launches"] > 0 and out["e2e"]["value"] > 0
    assert out["config"]["model"] == "vit_b_16" and out["config"]["cuda_graph"] is True


def test_imagenet_trainer_vit_b_32(tmp_path):
    sys.path.insert(0, ROOT)
    import io

    from distributeddeeplearning_b200.cli import launcher

    out, err = io.StringIO(), io.StringIO()
    res = launcher.launch("distributeddeeplearning_b200.workloads.imagenet",
                          ["--epochs", "1", "--batch_size", "16", "--model", "vit_b_32",
                           "--save_filepath", str(tmp_path / "ck-{epoch}.pt")], gpus=1, record=False, stdout=out,
                          stderr=err, timeout=900, env={"PYTHONPATH": ROOT, "FAKE_DATA_LENGTH": "64"})
    assert res.returncode == 0, (out.getvalue() + err.getvalue())[-3000:]
    assert "Training epoch 0 took" in out.getvalue()
