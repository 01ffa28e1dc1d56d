"""GPU tests (H100) of MNASNet: the `mnasnet` group of tools/gpu_diag.py (a native-only training step of each width,
mnasnet1_0 against torchvision, graph replay), its layer checks under the forced persistent / CTA-pair conv kernels and
the benchmark entry point under graph capture."""
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


def test_mnasnet_group():
    _group("mnasnet")


def test_mnasnet_layers_persistent_forced():
    _group("mnasnet_layers", env={"DDL_CONV_PERSISTENT": "2", "DDL_CONV_DEEP": "0", "DDL_CONV_AUTOTUNE": "0"})


def test_mnasnet_layers_cluster_pairs():
    _group("mnasnet_layers", env={"DDL_CONV_CLUSTER": "1", "DDL_CONV_PERSISTENT": "2"})


def test_bench_mnasnet1_0():
    r = subprocess.run([sys.executable, os.path.join(ROOT, "bench.py"), "--model", "mnasnet1_0", "--steps", "3",
                        "--warmup", "3"], cwd=ROOT, capture_output=True, text=True, timeout=900)
    assert r.returncode == 0, (r.stdout + r.stderr)[-3000:]
    out = json.loads([l for l in r.stdout.splitlines() if l.startswith("{")][-1])
    assert out["value"] > 0 and out["gpu_launches"] > 0 and out["e2e"]["value"] > 0
    assert out["config"]["cuda_graph"] is True and out["config"]["model"] == "mnasnet1_0"
