"""GPU tests (H100) of the device augmentation path: the `augment` group of tools/gpu_diag.py (the resized-crop kernel
against its float64 twin, bitwise repeatability, channel 3, a loader batch against the host PIL path), and the two
ImageNet trainers with --augment device on a generated JPEG folder: imagenet.py on class folders and on record shards,
one epoch with validation and the step captured into a CUDA graph, and hvd_imagenet.py for one epoch."""
import io
import os
import subprocess
import sys

import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
pytestmark = pytest.mark.gpu


def test_augment_group():
    r = subprocess.run([sys.executable, os.path.join(ROOT, "tools", "gpu_diag.py"), "--group", "augment"], cwd=ROOT,
                       capture_output=True, text=True, timeout=1800)
    out = r.stdout + r.stderr
    tail = "\n".join(l for l in out.splitlines() if "FAIL" in l or "Error" in l)[:3000] + "\n...\n" + out[-3000:]
    assert r.returncode == 0, tail
    assert "FAIL" not in r.stdout, tail


@pytest.fixture(scope="module")
def folders(tmp_path_factory):
    sys.path.insert(0, os.path.join(ROOT, "tools"))
    sys.path.insert(0, ROOT)
    from augment_bench import make_folder

    from distributeddeeplearning_b200.data import records

    base = tmp_path_factory.mktemp("augment")
    train = make_folder(str(base / "train"), 64, seed=1)
    val = make_folder(str(base / "validation"), 32, seed=2)
    rec = {}
    for split, root in (("train", train), ("validation", val)):
        files, labels, _ = records.find_image_files(root)
        rec[split] = str(base / "records" / split)
        records.write_shards(files, labels, rec[split], split, 2)
    return {"train": train, "val": val, "rec_train": rec["train"], "rec_val": rec["validation"], "base": base}


def _launch(module, argv, cwd):
    from distributeddeeplearning_b200.cli import launcher

    out, err = io.StringIO(), io.StringIO()
    res = launcher.launch(module, argv, gpus=1, record=False, stdout=out, stderr=err, timeout=900,
                          env={"PYTHONPATH": ROOT, "DDL_LOG_DIR": os.path.join(cwd, "logs"), "DDL_RUN_DIR": cwd})
    log = out.getvalue() + err.getvalue()
    assert res.returncode == 0, log[-3000:]
    return log


@pytest.mark.parametrize("data_type", ["images", "records"])
def test_imagenet_trainer_device_augment(folders, data_type, tmp_path):
    train, val = ((folders["train"], folders["val"]) if data_type == "images"
                  else (folders["rec_train"], folders["rec_val"]))
    log = _launch("distributeddeeplearning_b200.workloads.imagenet",
                  ["--epochs", "1", "--batch_size", "16", "--use_gpu", "True", "--training_data_path", train,
                   "--validation_data_path", val, "--data_type", data_type, "--augment", "device", "--num_workers", "2"],
                  str(tmp_path))
    assert "training step captured into a CUDA graph" in log, log[-3000:]
    assert "Training epoch 0 took" in log, log[-3000:]
    assert log.count("total-samples:") >= 2, log[-3000:]          # the first train and the first validation batch


def test_hvd_trainer_device_augment(folders, tmp_path):
    log = _launch("distributeddeeplearning_b200.workloads.hvd_imagenet",
                  ["--epochs", "1", "--batch-size", "16", "--val-batch-size", "16", "--train-dir", folders["train"],
                   "--val-dir", folders["val"], "--augment", "device", "--num-workers", "2",
                   "--log-dir", str(tmp_path / "logs"), "--checkpoint-format", str(tmp_path / "ck-{epoch}.pth.tar")],
                  str(tmp_path))
    assert os.path.isfile(tmp_path / "ck-1.pth.tar"), log[-3000:]


def test_capture_beside_a_pinning_thread():
    """The trainers capture their step while the DataLoader's pin-memory thread keeps pinning new batches; with
    capture_error_mode="thread_local" the capture succeeds, the other thread's cudaHostAlloc calls succeed, and the
    graph replays the step."""
    sys.path.insert(0, ROOT)
    import threading

    import torch

    from distributeddeeplearning_b200.workloads.graph_step import GraphedStep

    def fn(x):
        for _ in range(200):              # a capture of some length, so the pinning thread runs during it
            x = x * 1.0001 + 0.5
        return x

    x = torch.arange(4096, dtype=torch.float32, device="cuda")
    stop, started, errors, pinned = threading.Event(), threading.Event(), [], [0]

    def pin():
        started.set()
        n = 1 << 16
        try:
            while not stop.is_set():
                torch.empty(n, dtype=torch.uint8).pin_memory()        # a new size each time: a fresh cudaHostAlloc
                pinned[0] += 1
                n += 4096
        except Exception as e:  # noqa: BLE001
            errors.append(repr(e))

    t = threading.Thread(target=pin)
    t.start()
    started.wait()
    try:
        g = GraphedStep(fn, None, capture_error_mode="thread_local")
        ok = g.capture((x,), warmup=1)
    finally:
        stop.set()
        t.join()
    assert ok and not g.failed and not errors, errors
    assert pinned[0] > 0
    y = torch.randn(4096, device="cuda")
    torch.testing.assert_close(g(y), fn(y), rtol=1e-5, atol=1e-5)
