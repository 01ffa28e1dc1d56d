"""Resume-capable ImageNet trainer — parity with the reference's orphan
``PyTorch_hvd/src/imagenet_pytorch_horovod.py`` (the upstream Horovod ResNet-50 example; call stack
SURVEY.md 3.4).

Same argparse flags (``:15-47``), checkpoint-per-epoch + resume scan + epoch broadcast
(``:62-72,228-235``), rank-0 restore then parameter / optimizer-state broadcast (``:135-144``),
SGD(momentum, wd) at ``base_lr * size`` with the warm-up / step schedule (``:122-123,206-219``),
cross-rank averaged ``Metric`` (``:239-251``), TensorBoard scalars ``train/loss|accuracy``,
``val/loss|accuracy`` (``:172-174,197-199``) and tqdm bars on rank 0 (``:152-170``).

Additions: ``--train-dir`` may be omitted to train on synthetic data (the reference script has no
data-free mode); ``--model``; ``--synthetic-length``.
"""
from __future__ import annotations

import argparse
import os
import sys

import torch

from .. import models, ops
from ..data import DeviceSyntheticLoader, FakeData, get_sampler
from ..parallel import Compression, DistributedOptimizer, dist
from ..utils.checkpoint import agreed_resume_epoch, load_checkpoint, save_checkpoint
from ..utils.lr_schedule import learning_rate
from ..utils.meters import Metric, top1_accuracy
from ..utils.runs import summary_writer


def build_parser():
    p = argparse.ArgumentParser(description="PyTorch ImageNet Example (b200-ddl)",
                                formatter_class=argparse.ArgumentDefaultsHelpFormatter)
    p.add_argument("--train-dir", default=None, help="path to training data (omit for synthetic data)")
    p.add_argument("--val-dir", default=None, help="path to validation data")
    p.add_argument("--log-dir", default="./logs", help="tensorboard log directory")
    p.add_argument("--checkpoint-format", default="./checkpoint-{epoch}.pth.tar", help="checkpoint file format")
    p.add_argument("--fp16-allreduce", action="store_true", default=False, help="use 16-bit compression during allreduce")
    p.add_argument("--batch-size", type=int, default=32, help="input batch size for training")
    p.add_argument("--val-batch-size", type=int, default=32, help="input batch size for validation")
    p.add_argument("--epochs", type=int, default=90, help="number of epochs to train")
    p.add_argument("--base-lr", type=float, default=0.0125, help="learning rate for a single GPU")
    p.add_argument("--warmup-epochs", type=float, default=5, help="number of warmup epochs")
    p.add_argument("--momentum", type=float, default=0.9, help="SGD momentum")
    p.add_argument("--wd", type=float, default=0.00005, help="weight decay")
    p.add_argument("--no-cuda", action="store_true", default=False, help="disables CUDA training")
    p.add_argument("--seed", type=int, default=42, help="random seed")
    p.add_argument("--model", default="resnet50")
    p.add_argument("--synthetic-length", type=int, default=int(os.getenv("FAKE_DATA_LENGTH", 1281167)))
    p.add_argument("--num-workers", type=int, default=4)
    p.add_argument("--precision", choices=["bf16", "fp8"], default="bf16",
                   help="tensor-core operand format of the forward / data-gradient convolutions (ops/fp8.py)")
    p.add_argument("--no-cuda-graph", action="store_true", default=False,
                   help="launch every kernel of the training step eagerly instead of replaying a captured CUDA graph")
    return p


def _progress(total, desc, disable):
    try:
        from tqdm import tqdm

        return tqdm(total=total, desc=desc, disable=disable)
    except Exception:  # pragma: no cover
        class _N:
            def __enter__(self): return self
            def __exit__(self, *a): return False
            def update(self, n): pass
            def set_postfix(self, *a, **k): pass
        return _N()


def main(argv=None) -> int:
    args = build_parser().parse_args(argv)
    if args.precision == "fp8":
        if args.no_cuda:
            raise SystemExit("--precision fp8 needs CUDA")
        from ..ops import fp8

        fp8.enable(True)
    args.cuda = not args.no_cuda and torch.cuda.is_available()
    if not args.cuda:
        os.environ["DDL_NO_CUDA"] = "1"
    dist.init()
    torch.manual_seed(args.seed)
    device = torch.device("cuda", torch.cuda.current_device()) if args.cuda else torch.device("cpu")
    if args.cuda:
        torch.cuda.manual_seed(args.seed)
    world, rank = dist.size(), dist.rank()
    verbose = rank == 0

    # resume: newest existing checkpoint, rank 0's answer wins
    resume_from_epoch = agreed_resume_epoch(args.checkpoint_format, args.epochs, root_rank=0)
    writer = summary_writer(args.log_dir) if verbose else None

    net = models.get_model(args.model)
    size, classes = models.input_size(net), getattr(net, "num_classes", 1000)
    prepare = None
    val_loader = None
    if args.train_dir is None:
        if args.cuda:
            train_loader = DeviceSyntheticLoader(args.synthetic_length, args.batch_size, size, classes, device, rank,
                                                 world, args.seed)
            train_sampler = train_loader
        else:
            ds = FakeData(n_classes=classes, dim=(size, size), length=args.synthetic_length,
                          data_transform=torch.FloatTensor)
            train_sampler = get_sampler(ds)
            train_loader = torch.utils.data.DataLoader(ds, batch_size=args.batch_size, sampler=train_sampler)
    else:
        from ..data.images import DeviceNormalizer, image_folder_loader

        train_loader, train_sampler = image_folder_loader(args.train_dir, args.batch_size, True, size,
                                                          args.num_workers, device_normalize=args.cuda)
        prepare = DeviceNormalizer(device) if args.cuda else None
        if args.val_dir:
            val_loader, _ = image_folder_loader(args.val_dir, args.val_batch_size, False, size, args.num_workers,
                                                device_normalize=args.cuda)
    if args.cuda:
        net.cuda()
    # Horovod: scale learning rate by the number of GPUs
    optimizer = torch.optim.SGD(net.parameters(), lr=args.base_lr * world, momentum=args.momentum,
                                weight_decay=args.wd)
    compression = Compression.fp16 if args.fp16_allreduce else Compression.none
    optimizer = DistributedOptimizer(optimizer, named_parameters=net.named_parameters(), compression=compression)

    if resume_from_epoch > 0:
        load_checkpoint(args.checkpoint_format.format(epoch=resume_from_epoch), net, optimizer, root_rank=0)
    else:
        if hasattr(optimizer, "broadcast_parameters"):
            dist.broadcast_parameters({k: v for k, v in net.named_buffers()}, root_rank=0)
        else:
            dist.broadcast_parameters(net.state_dict(), root_rank=0)
        dist.broadcast_optimizer_state(optimizer, root_rank=0)

    def criterion(output, target):
        return ops.aux_classification_loss(output, target, classes, getattr(net, "aux_loss_weight", None))

    carry = hasattr(optimizer, "piggyback")

    def train_step(data, target):
        """One optimisation step; returns (loss, accuracy) — cross-rank means when the fused engine carries them."""
        optimizer.zero_grad()
        output = net(data)
        loss = criterion(output, target)
        main_out = output[0] if isinstance(output, tuple) else output
        acc = top1_accuracy(main_out.detach()[:, :classes].float(), target)
        if carry:   # the reference's 2 blocking scalar allreduces per step ride in the last gradient bucket
            optimizer.piggyback(torch.stack([loss.detach().float(), acc.float()]))
        loss.backward()
        optimizer.step()
        if carry:
            avg = optimizer.averaged_scalars()
            return avg[0], avg[1]
        return loss.detach(), acc

    graph_state = {}

    def train(epoch):
        net.train()
        if hasattr(train_sampler, "set_epoch"):
            train_sampler.set_epoch(epoch)
        train_loss, train_acc = Metric("train_loss", device), Metric("train_accuracy", device)
        nb = len(train_loader)
        with _progress(nb, "Train Epoch     #{}".format(epoch + 1), not verbose) as t:
            for batch_idx, (data, target) in enumerate(train_loader):
                lr = learning_rate(args.base_lr, epoch, batch_idx, nb, world, args.warmup_epochs)
                for g in optimizer.param_groups:
                    g["lr"] = lr
                data, target = data.to(device, non_blocking=True), target.to(device, non_blocking=True)
                if prepare is not None:
                    data = prepare(data)
                if "step" not in graph_state:
                    from .graph_step import GraphedStep

                    graph_state["step"] = train_step
                    if not args.no_cuda_graph and GraphedStep.applicable(net, optimizer, data):
                        g = GraphedStep(train_step, optimizer)
                        if g.capture((data, target), warmup=2):
                            graph_state["step"] = g
                l, a = graph_state["step"](data, target)
                train_loss.update(l, averaged=carry)
                train_acc.update(a, averaged=carry)
                t.update(1)
        if writer:
            writer.add_scalar("train/loss", float(train_loss.avg), epoch)
            writer.add_scalar("train/accuracy", float(train_acc.avg), epoch)
        else:
            train_loss.avg, train_acc.avg      # collective: every rank takes part in the averaging

    @torch.no_grad()
    def validate(epoch):
        if val_loader is None:
            return
        net.eval()
        val_loss, val_acc = Metric("val_loss", device), Metric("val_accuracy", device)
        with _progress(len(val_loader), "Validate Epoch  #{}".format(epoch + 1), not verbose) as t:
            for data, target in val_loader:
                data, target = data.to(device, non_blocking=True), target.to(device, non_blocking=True)
                if prepare is not None:
                    data = prepare(data)
                output = net(data)
                val_loss.update(criterion(output, target))
                val_acc.update(top1_accuracy(output[:, :classes].float(), target))
                t.update(1)
        if writer:
            writer.add_scalar("val/loss", float(val_loss.avg), epoch)
            writer.add_scalar("val/accuracy", float(val_acc.avg), epoch)
        else:
            val_loss.avg, val_acc.avg

    for epoch in range(resume_from_epoch, args.epochs):
        train(epoch)
        validate(epoch)
        save_checkpoint(args.checkpoint_format.format(epoch=epoch + 1), net, optimizer, epoch=epoch + 1)
    if hasattr(optimizer, "check_errors"):
        optimizer.check_errors()
    if writer:
        writer.flush()
    dist.shutdown()
    return 0


if __name__ == "__main__":
    sys.exit(main())
