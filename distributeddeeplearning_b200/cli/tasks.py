"""PyInvoke task tree — the reference's control-plane CLI (``tasks.py:180-225``; listing
``README.md:272-310``) re-targeted from AzureML to this box.

    inv pytorch-benchmark.submit.local.synthetic
    inv pytorch-benchmark.submit.remote.synthetic --node-count 8
    inv pytorch-imagenet.submit.remote.synthetic --node-count 8 --epochs 1
    inv pytorch-imagenet.submit.local.images --epochs 1
    inv pytorch-hvd.submit.remote.synthetic --node-count 4
    inv tf-benchmark.submit.remote.synthetic --node-count 8        (TensorFlow twins collapse onto PyTorch)
    inv storage.prepare-imagenet / storage.image.upload-data / runs / experiments / tensorboard ...

Mapping (SURVEY.md 2.8): ``local`` = exactly one non-distributed rank (reference
``aml_compute.py:434-445``); ``remote --node-count N`` = N ranks, one per GPU of this box
(reference: N nodes x 4 ranks under MPI).  Script parameters are the reference's
(``--model resnet50 --batch-size 64`` for the benchmark, ``pytorch_benchmark.py:21-29``;
``--epochs N --use_gpu True`` for the trainer, ``pytorch_imagenet.py:23-31``).
"""
from __future__ import annotations

import json
import os
import sys

from invoke import Collection, task

from ..utils import config as cfg
from ..utils import runs as runs_mod
from . import launcher

_BENCH = "distributeddeeplearning_b200.workloads.benchmark"
_IMAGENET = "distributeddeeplearning_b200.workloads.imagenet"
_HVD = "distributeddeeplearning_b200.workloads.hvd_imagenet"


def _env():
    return cfg.load_config()


def _max_nodes() -> int:
    return int(_env().get("CLUSTER_MAX_NODES", 8))


def _submit(module, argv, gpus, experiment, no_cuda=False, env=None):
    res = launcher.launch(module, argv, gpus=gpus, no_cuda=no_cuda, experiment=experiment, env=env)
    print(res)
    if res.returncode != 0:
        sys.exit(res.returncode)
    return res


# ------------------------------------------------------------------ pytorch-benchmark
@task(help={"no_cuda": "CPU/gloo plumbing mode", "model": "torchvision model name", "batch_size": "per-GPU batch"})
def benchmark_local(c, model="resnet50", batch_size=64, no_cuda=False, eager=False):
    """Submit the synthetic benchmark for local execution (one rank)."""
    argv = ["--model", model, "--batch-size", str(batch_size)] + (["--no-cuda"] if no_cuda else [])
    argv += [] if (eager or no_cuda) else ["--cuda-graph"]     # batch 64 is launch-bound: replay the step from a graph
    _submit(_BENCH, argv, 1, "synthetic_benchmark_local", no_cuda)


@task(help={"node_count": "number of ranks (GPUs of this box)"})
def benchmark_remote(c, node_count=None, model="resnet50", batch_size=64, no_cuda=False, fp16_allreduce=False,
                     eager=False):
    """Submit the synthetic benchmark on --node-count ranks."""
    n = int(node_count or _max_nodes())
    argv = ["--model", model, "--batch-size", str(batch_size)]
    argv += ["--no-cuda"] if no_cuda else ([] if eager else ["--cuda-graph"])
    argv += ["--fp16-allreduce"] if fp16_allreduce else []
    _submit(_BENCH, argv, n, "synthetic_benchmark_remote", no_cuda)


# ------------------------------------------------------------------ pytorch-imagenet
def _imagenet_argv(epochs, use_gpu, train=None, val=None, extra=()):
    argv = ["--epochs", str(epochs), "--use_gpu", "True" if use_gpu else "False"]
    if train:
        argv += ["--training_data_path", train]
    if val:
        argv += ["--validation_data_path", val]
    return argv + list(extra)


def _trainer_extra(batch_size, precision, fp16_allreduce=False):
    extra = []
    if batch_size:
        extra += ["--batch_size", str(batch_size)]
    if precision and precision != "bf16":
        extra += ["--precision", str(precision)]
    if fp16_allreduce:
        extra += ["--fp16_allreduce", "True"]
    return extra


@task(help={"precision": "bf16 (default) or fp8 tensor-core operands", "batch_size": "per-GPU batch (script default 64)"})
def imagenet_synthetic_local(c, epochs=1, no_cuda=False, batch_size=None, precision="bf16"):
    """ImageNet trainer, synthetic data, one rank."""
    _submit(_IMAGENET, _imagenet_argv(epochs, not no_cuda, extra=_trainer_extra(batch_size, precision)), 1,
            "synthetic_images_local", no_cuda)


@task(help={"precision": "bf16 (default) or fp8 tensor-core operands", "batch_size": "per-GPU batch (script default 64)"})
def imagenet_synthetic_remote(c, node_count=None, epochs=1, no_cuda=False, batch_size=None, precision="bf16",
                              fp16_allreduce=False):
    """ImageNet trainer, synthetic data, --node-count ranks."""
    _submit(_IMAGENET, _imagenet_argv(epochs, not no_cuda, extra=_trainer_extra(batch_size, precision, fp16_allreduce)),
            int(node_count or _max_nodes()), "synthetic_images_remote", no_cuda)


def _augment_extra(augment):
    return ["--augment", str(augment)] if augment and augment != "host" else []


_AUGMENT_HELP = {"augment": "host (default; PIL in the loader workers) or device (one GPU kernel after the copy)"}


@task(help=_AUGMENT_HELP)
def imagenet_images_local(c, epochs=1, no_cuda=False, augment="host"):
    """ImageNet trainer on $DATA/train and $DATA/validation, one rank."""
    data = _env()["DATA"]
    _submit(_IMAGENET, _imagenet_argv(epochs, not no_cuda, os.path.join(data, "train"), os.path.join(data, "validation"),
                                      _augment_extra(augment)), 1, "real_images_local", no_cuda)


@task(help=_AUGMENT_HELP)
def imagenet_images_remote(c, node_count=None, epochs=1, no_cuda=False, augment="host"):
    """ImageNet trainer on the datastore's train/validation folders, --node-count ranks."""
    store = _datastore_path()
    _submit(_IMAGENET, _imagenet_argv(epochs, not no_cuda, os.path.join(store, "train"), os.path.join(store, "validation"),
                                      _augment_extra(augment)), int(node_count or _max_nodes()), "real_images_remote",
            no_cuda)


@task(help=_AUGMENT_HELP)
def imagenet_records_local(c, epochs=1, no_cuda=False, augment="host"):
    """ImageNet trainer on the record shards under $DATA/records (reference: tf-imagenet ... tfrecords), one rank."""
    rec = os.path.join(_env()["DATA"], "records")
    _submit(_IMAGENET, _imagenet_argv(epochs, not no_cuda, os.path.join(rec, "train"), os.path.join(rec, "validation"),
                                      ["--data_type", "records", *_augment_extra(augment)]), 1, "records_local", no_cuda)


@task(help=_AUGMENT_HELP)
def imagenet_records_remote(c, node_count=None, epochs=1, no_cuda=False, augment="host"):
    """ImageNet trainer on the datastore's record shards, --node-count ranks (file-level sharding across ranks)."""
    rec = os.path.join(_datastore_path(), "records")
    _submit(_IMAGENET, _imagenet_argv(epochs, not no_cuda, os.path.join(rec, "train"), os.path.join(rec, "validation"),
                                      ["--data_type", "records", *_augment_extra(augment)]),
            int(node_count or _max_nodes()), "records_remote", no_cuda)


# ------------------------------------------------------------------ pytorch-hvd (orphan in the reference; wired here)
@task
def hvd_synthetic_local(c, epochs=1, batch_size=32, no_cuda=False):
    argv = ["--epochs", str(epochs), "--batch-size", str(batch_size)] + (["--no-cuda"] if no_cuda else [])
    _submit(_HVD, argv, 1, "hvd_synthetic_local", no_cuda)


@task
def hvd_synthetic_remote(c, node_count=None, epochs=1, batch_size=32, no_cuda=False):
    argv = ["--epochs", str(epochs), "--batch-size", str(batch_size)] + (["--no-cuda"] if no_cuda else [])
    _submit(_HVD, argv, int(node_count or _max_nodes()), "hvd_synthetic_remote", no_cuda)


@task(help=_AUGMENT_HELP)
def hvd_images_remote(c, node_count=None, epochs=90, batch_size=32, no_cuda=False, augment="host"):
    store = _datastore_path()
    argv = ["--epochs", str(epochs), "--batch-size", str(batch_size), "--train-dir", os.path.join(store, "train"),
            "--val-dir", os.path.join(store, "validation")] + (["--no-cuda"] if no_cuda else [])
    argv += _augment_extra(augment)
    _submit(_HVD, argv, int(node_count or _max_nodes()), "hvd_images_remote", no_cuda)


# ------------------------------------------------------------------ experiment template (reference: all raise)
def _template(name):
    @task(name=name)
    def t(c):
        """Template task: copy ``control/experiment_template`` and implement your own submit."""
        raise NotImplementedError("You need to modify this call before being able to use it "
                                  "(see distributeddeeplearning_b200/control/experiment_template/)")
    return t


# ------------------------------------------------------------------ storage (local datastore instead of Azure blob)
def _datastore_path() -> str:
    e = _env()
    root = e.get("DATASTORE_ROOT") or os.path.join(os.getcwd(), e.get("DATASTORE_NAME", "datastore"))
    return root


@task
def create_resource_group(c):
    """Create the root that holds run history and datastores (reference: `az group create`)."""
    e = _env()
    for d in (e.get("RUNS_DIR", "runs"), os.path.dirname(_datastore_path()) or "."):
        os.makedirs(d, exist_ok=True)
    print("resource root ready")


@task(pre=[create_resource_group])
def create_premium_storage(c):
    """Reserve the datastore location (reference: BlockBlobStorage Premium_LRS account)."""
    os.makedirs(_datastore_path(), exist_ok=True)
    print("storage:", _datastore_path())


@task(pre=[create_premium_storage])
def store_key(c):
    """Persist the datastore location in .env (reference writes ACCOUNT_KEY with set_key)."""
    path = cfg.find_dotenv() or ".env"
    cfg.set_key(path, "DATASTORE_ROOT", os.path.abspath(_datastore_path()))
    print(f"DATASTORE_ROOT stored in {path}")


@task
def create_container(c):
    """Create the local datastore directory (reference: resource group -> storage account -> container)."""
    p = _datastore_path()
    os.makedirs(p, exist_ok=True)
    print("datastore:", p)


def _copy_tree(src, dst):
    import shutil

    if not os.path.isdir(src):
        raise SystemExit(f"{src} does not exist")
    os.makedirs(dst, exist_ok=True)
    shutil.copytree(src, dst, dirs_exist_ok=True)
    print(f"copied {src} -> {dst}")


@task(pre=[create_container])
def upload_training_data(c):
    _copy_tree(os.path.join(_env()["DATA"], "train"), os.path.join(_datastore_path(), "train"))


@task(pre=[create_container])
def upload_validation_data(c):
    _copy_tree(os.path.join(_env()["DATA"], "validation"), os.path.join(_datastore_path(), "validation"))


@task(pre=[upload_training_data, upload_validation_data])
def upload_data(c):
    """Upload train + validation folders to the datastore."""


@task
def download_training_data(c):
    _copy_tree(os.path.join(_datastore_path(), "train"), os.path.join(_env()["DATA"], "train"))


@task
def download_validation_data(c):
    _copy_tree(os.path.join(_datastore_path(), "validation"), os.path.join(_env()["DATA"], "validation"))


@task(pre=[download_training_data, download_validation_data])
def download_data(c):
    """Download train + validation folders from the datastore."""


@task
def prepare_imagenet(c, download_dir=None, target_dir=None, check_sha1=True):
    """Un-tar ILSVRC2012 train / validation archives into class folders (reference scripts/prepare_imagenet.py)."""
    from ..data import prepare_imagenet as prep

    e = _env()
    prep.main(download_dir or e["DATA"], target_dir or e["DATA"], check_sha1)


@task
def upload_records(c):
    """Copy the record shards to the datastore (reference: storage.tfrecords.upload-data via azcopy)."""
    _copy_tree(os.path.join(_env()["DATA"], "records"), os.path.join(_datastore_path(), "records"))


@task
def download_records(c):
    """Copy the record shards from the datastore (reference: storage.tfrecords.download-data)."""
    _copy_tree(os.path.join(_datastore_path(), "records"), os.path.join(_env()["DATA"], "records"))


@task
def generate_records(c, data_dir=None, output_dir=None, shards_train=1014, shards_val=128):
    """Convert class folders into sharded record files (reference: TFRecord converter, 1014/128 shards)."""
    from ..data import records

    e = _env()
    d = data_dir or e["DATA"]
    records.convert(d, output_dir or os.path.join(d, "records"), int(shards_train), int(shards_val))


# ------------------------------------------------------------------ workspace-level tasks
@task
def setup(c, path=".env"):
    """Write the .env template (reference: login + storage + upload; cookiecutter post-gen moves _dotenv_template)."""
    if os.path.exists(path):
        print(f"{path} exists; leaving it unchanged")
    else:
        print("wrote", cfg.write_env_template(path))
    create_container(c)


@task
def login(c):
    """No cloud account is needed on a local box; prints the detected devices instead."""
    try:
        import torch

        n = torch.cuda.device_count()
        print(f"{n} CUDA device(s): " + ", ".join(torch.cuda.get_device_name(i) for i in range(n)))
    except Exception as e:  # pragma: no cover
        print("torch unavailable:", e)


@task
def select_subscription(c, gpus=None):
    """Pin the maximum number of ranks (reference: pick the Azure subscription and persist it with set_key)."""
    path = cfg.find_dotenv() or ".env"
    if gpus is None:
        print("current CLUSTER_MAX_NODES =", _env().get("CLUSTER_MAX_NODES"))
        return
    cfg.set_key(path, "CLUSTER_MAX_NODES", str(int(gpus)))
    print(f"set CLUSTER_MAX_NODES={gpus} in {path}")


@task
def experiments(c):
    """List experiments of the local run history."""
    root = _env().get("RUNS_DIR", "runs")
    for e in runs_mod.list_experiments(root):
        print(e)


@task(help={"experiment": "experiment name", "last": "only the N most recent runs"})
def runs(c, experiment, last=None):
    """List runs of an experiment."""
    root = _env().get("RUNS_DIR", "runs")
    for r in runs_mod.list_runs(experiment, root, int(last) if last else None):
        print(json.dumps({k: r.get(k) for k in ("id", "status", "started", "ended", "world_size", "exit_code", "tags")}))


@task
def tensorboard(c, experiment, runs=None, port=6006):
    """Start TensorBoard on an experiment's run directories (reference: azureml.tensorboard on running runs)."""
    root = os.path.join(_env().get("RUNS_DIR", "runs"), experiment)
    logdir = root if runs is None else ",".join(os.path.join(root, r, "tb") for r in str(runs).split(","))
    c.run(f"{sys.executable} -m tensorboard.main --logdir {logdir} --port {port} --bind_all", pty=False)


@task
def delete(c, experiment=None):
    """Delete the run history of an experiment (reference: delete the resource group)."""
    import shutil

    root = _env().get("RUNS_DIR", "runs")
    target = os.path.join(root, experiment) if experiment else root
    shutil.rmtree(target, ignore_errors=True)
    print("removed", target)


@task(name="interactive", aliases=("i",))
def interactive(c):
    """Open an interactive Python session with the package imported."""
    c.run(f"{sys.executable} -i -c 'import distributeddeeplearning_b200 as ddl; print(ddl.__doc__)'", pty=True)


@task
def new_project(c, name="b200_ddl_project", path=".", experiment_name="experiment"):
    """Render a project skeleton (the cookiecutter generator of the reference)."""
    from ..control import template

    print("created", template.render_project(os.path.join(path, name), project_name=name, experiment_name=experiment_name))


# ------------------------------------------------------------------ namespace assembly
def _submit_collection(name, local=None, remote=None):
    sub = Collection("submit")
    if local:
        lc = Collection("local")
        for n, t in local.items():
            lc.add_task(t, n)
        sub.add_collection(lc)
    if remote:
        rc = Collection("remote")
        for n, t in remote.items():
            rc.add_task(t, n)
        sub.add_collection(rc)
    col = Collection(name)
    col.add_collection(sub)
    return col


# template type (cookiecutter ``type`` variable, ``cookiecutter.json:18-26``) -> the workload collections it keeps; the
# reference's post-gen hook was meant to delete the other project directories (``hooks/post_gen_project.py:19-33``)
WORKLOAD_TYPES = {
    "pytorch_benchmark": ("pytorch_benchmark",),
    "pytorch_imagenet": ("pytorch_imagenet",),
    "pytorch_hvd": ("pytorch_hvd",),
    "pytorch_template": ("pytorch_experiment",),
    "tensorflow_benchmark": ("tf_benchmark",),
    "tensorflow_imagenet": ("tf_imagenet",),
    "tensorflow_template": ("tf_experiment",),
}


def enabled_workloads():
    """Collections the project keeps: ``ENABLED_WORKLOADS`` (process env, else the project's .env; written by
    ``control.template.render_project`` when ``_remove_unused_projects`` is set) — None = everything."""
    raw = os.environ.get("ENABLED_WORKLOADS")
    if raw is None:
        try:
            raw = cfg.load_config(required=False).get("ENABLED_WORKLOADS")
        except Exception:
            raw = None
    if not raw or raw.strip().lower() == "all":
        return None
    keep = set()
    for t in raw.replace(";", ",").split(","):
        t = t.strip()
        if t:
            keep.update(WORKLOAD_TYPES.get(t, (t,)))
    return keep


def build_namespace() -> Collection:
    ns = Collection(setup, login, select_subscription, experiments, runs, tensorboard, delete, interactive, new_project)
    keep = enabled_workloads()

    def add(col):
        if keep is None or str(col.name).replace("-", "_") in keep:
            ns.add_collection(col)

    add(_submit_collection("pytorch_benchmark", {"synthetic": benchmark_local}, {"synthetic": benchmark_remote}))
    add(_submit_collection("pytorch_imagenet",
                           {"synthetic": imagenet_synthetic_local, "images": imagenet_images_local,
                            "records": imagenet_records_local},
                           {"synthetic": imagenet_synthetic_remote, "images": imagenet_images_remote,
                            "records": imagenet_records_remote}))
    add(_submit_collection("pytorch_hvd", {"synthetic": hvd_synthetic_local},
                           {"synthetic": hvd_synthetic_remote, "images": hvd_images_remote}))
    add(_submit_collection("pytorch_experiment",
                           {"synthetic": _template("exp_local_synthetic"), "images": _template("exp_local_images")},
                           {"synthetic": _template("exp_remote_synthetic"), "images": _template("exp_remote_images")}))
    # TensorFlow twins collapse onto the PyTorch workloads (BASELINE.json north-star)
    add(_submit_collection("tf_benchmark", {"synthetic": benchmark_local}, {"synthetic": benchmark_remote}))
    add(_submit_collection("tf_imagenet",
                           {"synthetic": imagenet_synthetic_local, "images": imagenet_images_local,
                            "tfrecords": imagenet_records_local},
                           {"synthetic": imagenet_synthetic_remote, "images": imagenet_images_remote,
                            "tfrecords": imagenet_records_remote}))
    add(_submit_collection("tf_experiment",
                           {"synthetic": _template("tfexp_local_synthetic")},
                           {"synthetic": _template("tfexp_remote_synthetic")}))
    storage = Collection("storage")
    storage.add_task(create_resource_group, "create-resource-group")
    storage.add_task(create_premium_storage, "create-premium-storage")
    storage.add_task(store_key, "store-key")
    storage.add_task(create_container, "create-container")
    storage.add_task(prepare_imagenet, "prepare-imagenet")
    image = Collection("image")
    for n, t in {"upload-training-data": upload_training_data, "upload-validation-data": upload_validation_data,
                 "upload-data": upload_data, "download-training-data": download_training_data,
                 "download-validation-data": download_validation_data, "download-data": download_data,
                 "prepare-imagenet": prepare_imagenet}.items():
        image.add_task(t, n)
    storage.add_collection(image)
    rec = Collection("tfrecords")
    rec.add_task(generate_records, "generate-tf-records")
    rec.add_task(upload_records, "upload-data")
    rec.add_task(download_records, "download-data")
    storage.add_collection(rec)
    ns.add_collection(storage)
    return ns


namespace = build_namespace()
