"""GPU tests (H100) of MaxViT: the `maxvit` group of tools/gpu_diag.py (grid and window partition attention forward and
backward at every stage shape of maxvit_t at 224 and 448 and edge cases, bitwise-repeatable backward, Swin's window
kernel at MaxViT's shapes, BN-GELU, the tanh pair, maxvit_t against torchvision, graph replay and an fp8 session), the
benchmark entry point and the ImageNet trainer on maxvit_t."""
import json
import os
import subprocess
import sys

import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
pytestmark = pytest.mark.gpu


def test_maxvit_group():
    r = subprocess.run([sys.executable, os.path.join(ROOT, "tools", "gpu_diag.py"), "--group", "maxvit"], cwd=ROOT,
                       capture_output=True, text=True, timeout=1500)
    out = r.stdout + r.stderr
    tail = "\n".join(l for l in out.splitlines() if "FAIL" in l or "Error" in l)[:3000] + "\n...\n" + out[-3000:]
    assert r.returncode == 0, tail
    assert "FAIL" not in r.stdout, tail


def test_bench_maxvit_t():
    r = subprocess.run([sys.executable, os.path.join(ROOT, "bench.py"), "--model", "maxvit_t", "--steps", "3",
                        "--warmup", "3", "--batch-size", "32"], cwd=ROOT, capture_output=True, text=True, timeout=900)
    assert r.returncode == 0, (r.stdout + r.stderr)[-3000:]
    out = json.loads([l for l in r.stdout.splitlines() if l.startswith("{")][-1])
    for key in ("metric", "value", "unit", "n_gpus", "steps", "warmup", "ms_per_step", "higher_is_better", "scaling",
                "vs_baseline", "dtype", "data", "config", "clocks", "e2e", "gpu_launches"):
        assert key in out, key
    assert out["value"] > 0 and out["gpu_launches"] > 0 and out["e2e"]["value"] > 0
    assert out["config"]["model"] == "maxvit_t" and out["config"]["cuda_graph"] is True


def test_imagenet_trainer_maxvit_t(tmp_path):
    sys.path.insert(0, ROOT)
    import io

    from distributeddeeplearning_b200.cli import launcher

    out, err = io.StringIO(), io.StringIO()
    res = launcher.launch("distributeddeeplearning_b200.workloads.imagenet",
                          ["--epochs", "1", "--batch_size", "16", "--model", "maxvit_t",
                           "--save_filepath", str(tmp_path / "ck-{epoch}.pt")], gpus=1, record=False, stdout=out,
                          stderr=err, timeout=900, env={"PYTHONPATH": ROOT, "FAKE_DATA_LENGTH": "64"})
    assert res.returncode == 0, (out.getvalue() + err.getvalue())[-3000:]
    assert "Training epoch 0 took" in out.getvalue()
