"""GPU tests (H100) of the weight-gradient kernel (conv_wgrad_kernel through conv_wgrad / linear_wgrad): the `wgrad`
group of tools/gpu_diag.py (one subprocess per run, as in test_gpu.py), element-wise against float64 at training scale,
under the default policy and under each accepted operand-mode hook."""
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


def test_wgrad_group():
    """Default configuration: swapped 64-channel tiles for narrow outputs, TMA tile and stem modes."""
    _group("wgrad")


def test_wgrad_group_no_swap():
    """DDL_WGRAD_SWAP=0: every output-channel tile 128 wide, the narrow ones half empty."""
    _group("wgrad", env={"DDL_WGRAD_SWAP": "0"})


def test_wgrad_group_gather_modes():
    """The cp.async gather producers in place of the TMA tile windows (stride 1 and 2) and the TMA stem."""
    _group("wgrad", env={"DDL_DISABLE_TILE_TMA": "1", "DDL_DISABLE_TILE_S2": "1", "DDL_DISABLE_STEM_TMA": "1"})
