import os
import sys

import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
if ROOT not in sys.path:
    sys.path.insert(0, ROOT)

os.environ.setdefault("OMP_NUM_THREADS", "2")


def pytest_configure(config):
    config.addinivalue_line("markers", "gpu: needs a CUDA device (run on an H100 box with `pytest -m gpu`)")


def pytest_collection_modifyitems(config, items):
    try:
        import torch

        has_gpu = torch.cuda.is_available()
    except Exception:
        has_gpu = False
    if has_gpu:
        return
    skip = pytest.mark.skip(reason="no CUDA device")
    for item in items:
        if "gpu" in item.keywords:
            item.add_marker(skip)


@pytest.fixture(autouse=True)
def _few_threads():
    import torch

    torch.set_num_threads(2)
    yield


@pytest.fixture(autouse=True)
def _artefacts_outside_the_repo(tmp_path, monkeypatch):
    """Run history, TensorBoard event files and checkpoints of anything a test launches go to the test's tmp dir
    (child processes inherit the environment): the suite must not create or delete files inside the repository."""
    monkeypatch.setenv("DDL_RUNS_DIR", str(tmp_path / "runs"))
    monkeypatch.setenv("DDL_LOG_DIR", str(tmp_path / "logs"))
    yield
