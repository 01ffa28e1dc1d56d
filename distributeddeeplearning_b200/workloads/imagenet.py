"""ImageNet trainer with synthetic or real data — parity with the reference's
``PyTorch_imagenet/src/imagenet_pytorch_horovod.py`` (call stack SURVEY.md 3.3).

Same CLI (python-fire style ``main`` kwargs, ``:292-303``), env (``DISTRIBUTED``, ``EPOCHS``,
``FAKE_DATA_LENGTH``, ``LOG_CONFIG``), log lines (per-100-step ``" duration({})  loss:{}
total-samples: {}"`` ``:173,197``; ``"setting lr to ..."`` ``:289``; ``"Training epoch N took X
seconds"`` ``:416``; summary block ``:233-245``), TensorBoard scalars (``Train/Loss``, ``Train/Acc``,
``Train/BatchTime``, ``Validation/*`` ``:426-436``) and run-history rows (``:425,434``).

Deliberate fixes of reference bugs (SURVEY.md 2.9): the summary divides ALL epochs' images by ALL
epochs' time (Q3); checkpoints work on every rank and per epoch when the path has ``{epoch}`` (Q4);
validation runs under ``no_grad`` (Q5); metrics are accumulated on the device and read back every
``log_interval`` steps instead of three ``.item()`` syncs per step (K18).
"""
from __future__ import annotations

import logging
import os

import torch

from .. import models, ops
from ..data import DeviceSyntheticLoader, FakeData, get_sampler
from ..parallel import Compression, DistributedOptimizer, dist
from ..utils import Timer, logconf
from ..utils.checkpoint import save_checkpoint
from ..utils.firelite import Fire
from ..utils.lr_schedule import adjust_learning_rate
from ..utils.meters import AverageMeter
from ..utils.runs import Run, summary_writer

_WIDTH = _HEIGHT = 224
_LR = 0.001
_EPOCHS = os.getenv("EPOCHS", 5)
_BATCHSIZE = 64
_SEED = 42
_LOG_INTERVAL = 100


def _str_to_bool(s) -> bool:
    return "t" in str(s).lower()


def _data_length() -> int:
    return int(os.getenv("FAKE_DATA_LENGTH", 1281167))


def _log_summary(data_length, duration, batch_size, world):
    logger = logging.getLogger(__name__)
    logger.info("Data length:      {}".format(data_length))
    logger.info("Total duration:   {:.3f}".format(duration))
    logger.info("Total images/sec: {:.3f}".format(data_length / max(duration, 1e-9)))
    logger.info("Batch size:       (Per GPU {}: Total {})".format(batch_size, world * batch_size))
    logger.info("Distributed:      {}".format("True" if world > 1 else "False"))
    logger.info("Num GPUs:         {:.3f}".format(world))


class _DeviceMetrics:
    """loss / top-1 / top-5 accumulated on the device; one readback per log interval."""

    def __init__(self, device):
        self.loss_sum = torch.zeros((), dtype=torch.float32, device=device)
        self.correct = torch.zeros(2, dtype=torch.int64, device=device)
        self.samples = 0
        self.steps = 0

    def update(self, loss, output, target, classes):
        self.loss_sum += loss.detach().float()
        self.correct += ops.topk_correct(output.detach() if not isinstance(output, tuple) else output[0].detach(),
                                         target, classes).to(torch.int64)
        self.samples += int(target.shape[0])
        self.steps += 1

    def read(self):
        n = max(self.samples, 1)
        c = self.correct.tolist()
        return {"loss": float(self.loss_sum) / max(self.steps, 1), "acc": 100.0 * c[0] / n, "acc5": 100.0 * c[1] / n}


def _train_step_fn(model, criterion, optimizer):
    def step(data, target):
        optimizer.zero_grad()
        output = model(data)
        loss = criterion(output, target)
        loss.backward()
        optimizer.step()
        return loss.detach(), (output[0] if isinstance(output, tuple) else output).detach()
    return step


def train(train_loader, model, criterion, optimizer, base_lr, warmup_epochs, epoch, device, classes, world,
          prepare=None, graph=None):
    """One epoch.  ``graph``: an (initially empty) dict — when given, the training step is captured into a CUDA graph on
    the first full batch and replayed for every batch of that shape (``graph_step.GraphedStep``)."""
    logger = logging.getLogger(__name__)
    batch_time = AverageMeter()
    metrics = _DeviceMetrics(device)
    msg = " duration({})  loss:{} total-samples: {}"
    t = Timer().start()
    nb = len(train_loader)
    last_loss = None
    for i, (data, target) in enumerate(train_loader):
        adjust_learning_rate(optimizer, base_lr, warmup_epochs, nb, epoch, i, world, log=dist.rank() == 0)
        data, target = data.to(device, non_blocking=True), target.to(device, non_blocking=True)
        if prepare is not None:
            data = prepare(data)
        if graph is not None and "step" not in graph:
            from .graph_step import GraphedStep

            fn = _train_step_fn(model, criterion, optimizer)
            graph["step"] = fn
            if GraphedStep.applicable(model, optimizer, data):
                g = GraphedStep(fn, optimizer, logger.info)
                if g.capture((data, target), warmup=2):
                    graph["step"] = g
                    logger.info("training step captured into a CUDA graph (%d kernels per replay)" % g.launches)
        if graph is not None:
            loss, output = graph["step"](data, target)
        else:
            optimizer.zero_grad()
            output = model(data)
            loss = criterion(output, target)
            loss.backward()
            optimizer.step()
        metrics.update(loss, output, target, classes)
        last_loss = loss
        if i % _LOG_INTERVAL == 0:
            t.stop()
            batch_time.update(t.elapsed, n=_LOG_INTERVAL)
            logger.info(msg.format(t.elapsed, float(last_loss), i * int(target.shape[0])))
            if hasattr(optimizer, "check_errors"):
                optimizer.check_errors()          # a barrier timeout must stop the job before more steps / checkpoints
            t.start()
    out = metrics.read()
    out["batch_time"] = batch_time.avg
    return out


@torch.no_grad()
def validate(val_loader, model, criterion, device, classes, prepare=None):
    logger = logging.getLogger(__name__)
    metrics = _DeviceMetrics(device)
    msg = " duration({})  loss:{} total-samples: {}"
    t = Timer().start()
    for i, (data, target) in enumerate(val_loader):
        data, target = data.to(device, non_blocking=True), target.to(device, non_blocking=True)
        if prepare is not None:
            data = prepare(data)
        output = model(data)
        loss = criterion(output, target)
        metrics.update(loss, output, target, classes)
        if i % _LOG_INTERVAL == 0:
            logger.info(msg.format(t.elapsed, float(loss), i * int(target.shape[0])))
            t.start()
    return metrics.read()


def main(training_data_path=None, validation_data_path=None, use_gpu=False, save_filepath=None, model="resnet50",
         epochs=_EPOCHS, batch_size=_BATCHSIZE, fp16_allreduce=False, base_lr=0.0125, warmup_epochs=5,
         num_workers=5, host_data=False, cuda_graph=True, data_type=None, precision="bf16"):
    """``cuda_graph``: on a GPU with the fused engine, replay the training step from a captured CUDA graph (the
    reference's default batch of 64 per GPU is launch-bound: ~340 kernels per ResNet-50 step).
    ``data_type``: ``synthetic`` | ``images`` (class folders) | ``records`` / ``tfrecords`` (sharded record files
    written by ``inv storage.tfrecords.generate-tf-records``; the data paths are then the shard directories) — the
    switch of the reference's TF trainer tasks (``TensorFlow_imagenet/tensorflow_imagenet.py:110-151``).  Default:
    synthetic without a training path, images with one.
    ``precision``: ``bf16`` (default) or ``fp8`` — e4m3 / e5m2 tensor-core operands for the forward and data-gradient
    convolutions (``ops/fp8.py``; the analogue of the reference's ``--use_fp16``,
    ``TensorFlow_benchmark/tensorflow_benchmark.py:51``)."""
    logger = logging.getLogger(__name__)
    epochs = int(epochs)
    cuda_graph = _str_to_bool(cuda_graph) if isinstance(cuda_graph, str) else bool(cuda_graph)
    use_gpu = _str_to_bool(use_gpu) if isinstance(use_gpu, str) else bool(use_gpu)
    use_gpu = use_gpu and torch.cuda.is_available()
    if not use_gpu:
        os.environ["DDL_NO_CUDA"] = "1"
    dist.init()
    world, rank = dist.size(), dist.rank()
    device = torch.device("cuda", torch.cuda.current_device()) if use_gpu else torch.device("cpu")
    logger.info(f"Running on {device}")
    if world > 1:
        logger.info("Running Distributed")
    torch.manual_seed(_SEED)
    if use_gpu:
        torch.cuda.manual_seed(_SEED)
    logger.info("PyTorch version {}".format(torch.__version__))
    precision = str(precision).lower()
    if precision not in ("bf16", "fp8"):
        raise ValueError(f"precision must be bf16 or fp8, got {precision!r}")
    if precision == "fp8":
        if not use_gpu:
            raise ValueError("--precision fp8 needs --use_gpu True (fp8 tensor cores)")
        from ..ops import fp8

        fp8.enable(True)
        logger.info("Precision: fp8 operands (e4m3 activations/weights) for the forward convolutions, fp32 accumulate")

    run = writer = None
    if rank == 0:
        run = Run.get_context("pytorch_imagenet")
        run.tag("model", value=model)
        # the reference wipes and rewrites ./logs of the job's private working directory (``:324-329``); a local
        # run keeps its event files inside its own run directory instead (DDL_LOG_DIR overrides), so nothing in
        # the caller's cwd is deleted or littered
        logs_dir = os.getenv("DDL_LOG_DIR") or os.path.join(run.dir, "logs")
        writer = summary_writer(logs_dir)

    net = models.get_model(model)
    size = models.input_size(net)
    classes = getattr(net, "num_classes", 1000)
    prepare = None
    val_loader = None
    data_type = (data_type or ("synthetic" if training_data_path is None else "images")).lower()
    if data_type == "tfrecords":
        data_type = "records"
    if data_type not in ("synthetic", "images", "records"):
        raise ValueError(f"data_type must be synthetic, images or records, got {data_type!r}")
    if data_type != "synthetic" and training_data_path is None:
        raise ValueError(f"--data_type {data_type} needs --training_data_path")
    if data_type == "synthetic":
        logger.info("Setting up fake loaders")
        if use_gpu and not host_data:
            train_loader = DeviceSyntheticLoader(_data_length(), batch_size, size, classes, device, rank, world, _SEED)
            train_sampler = train_loader
        else:
            ds = FakeData(n_classes=classes, dim=(size, size), length=_data_length(), data_transform=torch.FloatTensor)
            train_sampler = get_sampler(ds)
            train_loader = torch.utils.data.DataLoader(ds, batch_size=batch_size, sampler=train_sampler,
                                                       num_workers=num_workers if use_gpu else 0, pin_memory=use_gpu)
    elif data_type == "records":
        from ..data.images import DeviceNormalizer
        from ..data.records import RecordLoader

        logger.info("Setting up record loaders")
        logger.info(f"Loading training shards from {training_data_path}")
        train_loader = RecordLoader(training_data_path, "train", batch_size, True, size, num_workers, rank, world,
                                    normalize_on_host=not use_gpu, seed=_SEED)
        train_sampler = train_loader
        prepare = DeviceNormalizer(device) if use_gpu else None
        if validation_data_path is not None:
            logger.info(f"Loading validation shards from {validation_data_path}")
            val_loader = RecordLoader(validation_data_path, "validation", batch_size, False, size, num_workers, rank,
                                      world, normalize_on_host=not use_gpu)
    else:
        from ..data.images import DeviceNormalizer, image_folder_loader

        logger.info("Setting up loaders")
        logger.info(f"Loading training from {training_data_path}")
        train_loader, train_sampler = image_folder_loader(training_data_path, batch_size, True, size, num_workers,
                                                          device_normalize=use_gpu)
        prepare = DeviceNormalizer(device) if use_gpu else None
        if validation_data_path is not None:
            logger.info(f"Loading validation from {validation_data_path}")
            val_loader, _ = image_folder_loader(validation_data_path, batch_size, False, size, num_workers,
                                                device_normalize=use_gpu)

    logger.info("Loading model")
    if use_gpu:
        net.cuda()
    optimizer = torch.optim.SGD(net.parameters(), lr=_LR * world, momentum=0.9)
    compression = Compression.fp16 if _str_to_bool(fp16_allreduce) else Compression.none
    optimizer = DistributedOptimizer(optimizer, named_parameters=net.named_parameters(), compression=compression)
    if hasattr(optimizer, "broadcast_parameters"):
        dist.broadcast_parameters({k: v for k, v in net.named_buffers()}, root_rank=0)
    else:
        dist.broadcast_parameters(net.state_dict(), root_rank=0)
    dist.broadcast_optimizer_state(optimizer, root_rank=0)

    def criterion(output, target):
        return ops.aux_classification_loss(output, target, classes, getattr(net, "aux_loss_weight", None))

    logger.info("Training ...")
    total_time = 0.0
    graph_state = {} if (cuda_graph and use_gpu) else None
    for epoch in range(epochs):
        with Timer(output=logger.info, prefix=f"Training epoch {epoch} ") as t:
            net.train()
            if hasattr(train_sampler, "set_epoch"):
                train_sampler.set_epoch(epoch)
            metrics = train(train_loader, net, criterion, optimizer, base_lr, warmup_epochs, epoch, device, classes,
                            world, prepare, graph=graph_state)
            if use_gpu:
                torch.cuda.synchronize()
        total_time += t.elapsed
        if rank == 0:
            run.log_row("Training metrics", epoch=epoch, **metrics)
            writer.add_scalar("Train/Loss", metrics["loss"], epoch)
            writer.add_scalar("Train/Acc", metrics["acc"], epoch)
            writer.add_scalar("Train/BatchTime", metrics["batch_time"], epoch)
        if val_loader is not None:
            net.eval()
            vm = validate(val_loader, net, criterion, device, classes, prepare)
            if rank == 0:
                run.log_row("Validation metrics", epoch=epoch, **vm)
                writer.add_scalar("Validation/Loss", vm["loss"], epoch)
                writer.add_scalar("Validation/Acc", vm["acc"], epoch)
        if save_filepath is not None:
            save_checkpoint(str(save_filepath).format(epoch=epoch + 1), net, optimizer, epoch=epoch + 1)
    if hasattr(optimizer, "check_errors"):
        optimizer.check_errors()
    per_rank = getattr(train_loader, "per_rank", None)
    seen = epochs * (per_rank * world if per_rank is not None else len(train_loader.dataset))
    if rank == 0:
        _log_summary(seen, total_time, batch_size, world)
        writer.flush()
        run.complete()
    dist.shutdown()
    return {"images": seen, "seconds": total_time}


def cli(argv=None):
    logconf.configure("imagenet")
    return Fire(main, argv)


if __name__ == "__main__":
    cli()
