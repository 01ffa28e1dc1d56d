"""Recipe for bench.py's `--impl reference` arm: copy the reference's workload scripts VERBATIM (byte-identical) into the
git-ignored oracle/_ref/, so that they run unmodified against baseline/hvd_shim (the reference's pinned horovod 0.15 /
torch 1.0 stack cannot be installed: the reference is a cookiecutter template without setup.py / pyproject.toml).

The reference is microsoft/DistributedDeepLearning, checked out next to this repository (../reference) or wherever
DDL_REFERENCE_ROOT points.  `build()` runs this; without a reference checkout it leaves oracle/_ref/ as it is (a tree
that already carries the scripts keeps them), and the reference arm reports itself unavailable.
"""
import json
import os
import shutil
import sys

HERE = os.path.dirname(os.path.abspath(__file__))
REF = os.environ.get("DDL_REFERENCE_ROOT", os.path.join(os.path.dirname(os.path.dirname(HERE)), "reference"))
DST = os.path.join(HERE, "_ref")
TEMPLATE = "{{cookiecutter.project_name}}"
SCRIPTS = ["PyTorch_benchmark/src/pytorch_synthetic_benchmark.py",
           "PyTorch_imagenet/src/imagenet_pytorch_horovod.py", "PyTorch_imagenet/src/timer.py",
           "PyTorch_imagenet/src/logging.conf", "PyTorch_hvd/src/imagenet_pytorch_horovod.py",
           "PyTorch_hvd/src/timer.py", "PyTorch_hvd/src/logging.conf"]
BENCH_SCRIPT = os.path.join(DST, SCRIPTS[0])


def build() -> dict:
    record = {"reference_root": REF}
    if not os.path.isdir(os.path.join(REF, TEMPLATE)):
        record["status"] = "no reference checkout; oracle/_ref left as it is"
        record["available"] = os.path.isfile(BENCH_SCRIPT)
        return record
    copied = []
    for rel in SCRIPTS:
        src = os.path.join(REF, TEMPLATE, rel)
        if os.path.isfile(src):
            dst = os.path.join(DST, rel)
            os.makedirs(os.path.dirname(dst), exist_ok=True)
            shutil.copyfile(src, dst)
            copied.append(rel)
    record["copied_verbatim"] = copied
    record["status"] = "scripts copied verbatim"
    record["available"] = os.path.isfile(BENCH_SCRIPT)
    with open(os.path.join(DST, "INSTALL.json"), "w") as f:
        json.dump(record, f, indent=1)
    return record


if __name__ == "__main__":
    print(json.dumps(build()))
    sys.exit(0)
