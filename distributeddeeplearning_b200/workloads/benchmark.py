"""Synthetic training benchmark — same flags and rank-0 stdout as the reference's
``PyTorch_benchmark/src/pytorch_synthetic_benchmark.py`` (flags ``:14-48``, output ``:101-126``):

    Model: resnet50
    Batch size: 64
    Number of GPUs: 8
    Running warmup...
    Running benchmark...
    Iter #0: 123.4 img/sec per GPU
    Img/sec per GPU: 123.4 +-5.6
    Total img/sec on 8 GPU(s): 987.2 +-44.8

What differs underneath (SURVEY.md 3.2): the step is device-timed with CUDA events and reduced
with max over ranks (the reference host-times rank 0 with ``timeit`` and no synchronize); the model
runs the hand-written sm_90a kernels in bf16 with fp32 master weights; ``DistributedOptimizer``
is the fused NVLink allreduce+SGD engine; the fixed batch is generated on the device.
"""
from __future__ import annotations

import argparse
import json
import sys
from typing import Dict, List, Optional

import numpy as np
import torch

from .. import models, ops
from ..data import fixed_synthetic_batch
from ..parallel import Compression, DistributedOptimizer, dist
from ..utils.faults import maybe_inject


def build_parser() -> argparse.ArgumentParser:
    p = argparse.ArgumentParser(description="PyTorch Synthetic Benchmark (b200-ddl)",
                                formatter_class=argparse.ArgumentDefaultsHelpFormatter)
    p.add_argument("--fp16-allreduce", action="store_true", default=False,
                   help="use 16-bit compression during allreduce (bf16 on the NVLink wire)")
    p.add_argument("--model", type=str, default="resnet50", help="model to benchmark")
    p.add_argument("--batch-size", type=int, default=32, help="input batch size")
    p.add_argument("--num-warmup-batches", type=int, default=10,
                   help="number of warm-up batches that don't count towards benchmark")
    p.add_argument("--num-batches-per-iter", type=int, default=10, help="number of batches per benchmark iteration")
    p.add_argument("--num-iters", type=int, default=10, help="number of benchmark iterations")
    p.add_argument("--no-cuda", action="store_true", default=False, help="disables CUDA training")
    # additions (not in the reference)
    p.add_argument("--lr", type=float, default=0.01, help="SGD learning rate (reference: 0.01, no momentum)")
    p.add_argument("--momentum", type=float, default=0.0)
    p.add_argument("--json", type=str, default=None, help="also write a JSON summary to this path ('-' = stdout)")
    p.add_argument("--profile", action="store_true", help="wrap phases in NVTX ranges")
    p.add_argument("--precision", choices=["bf16", "fp8"], default="bf16",
                   help="tensor-core operand format of the forward / data-gradient convolutions")
    p.add_argument("--phase-times", action="store_true",
                   help="after the benchmark, device-time forward / backward / optimizer join of a few eager steps and "
                        "the per-bucket allreduce+SGD kernels (per-phase profile; reference has none)")
    p.add_argument("--cuda-graph", action="store_true",
                   help="capture the training step into a CUDA graph after warm-up and replay it (small batches are "
                        "launch-bound: ~340 kernels per ResNet-50 step)")
    return p


def log(s: str, nl: bool = True) -> None:
    if dist.rank() != 0:
        return
    print(s, end="\n" if nl else "", flush=True)


class BenchmarkSession:
    """Model + optimizer + fixed batch; ``step()`` is one full training iteration."""

    def __init__(self, model_name: str, batch_size: int, cuda: bool, fp16_allreduce: bool = False, lr: float = 0.01,
                 momentum: float = 0.0, seed: int = 0, profile: bool = False, data_seed_offset: Optional[int] = None):
        self.cuda = cuda
        self.profile = bool(profile) and cuda
        self.device = torch.device("cuda", torch.cuda.current_device()) if cuda else torch.device("cpu")
        torch.manual_seed(seed)
        self.model = models.get_model(model_name)
        self.model.train()
        if cuda:
            self.model.cuda()
        self.num_classes = getattr(self.model, "num_classes", 1000)
        opt = torch.optim.SGD(self.model.parameters(), lr=lr, momentum=momentum)
        compression = Compression.fp16 if fp16_allreduce else Compression.none
        self.optimizer = DistributedOptimizer(opt, named_parameters=self.model.named_parameters(),
                                              compression=compression)
        if not hasattr(self.optimizer, "broadcast_parameters"):
            dist.broadcast_parameters(self.model.state_dict(), root_rank=0)
            dist.broadcast_optimizer_state(self.optimizer, root_rank=0)
        else:
            dist.broadcast_parameters({k: v for k, v in self.model.named_buffers()}, root_rank=0)
            dist.broadcast_optimizer_state(self.optimizer, root_rank=0)
        size = models.input_size(self.model)
        # every rank draws its OWN fixed batch (the reference draws unseeded per-process data,
        # pytorch_synthetic_benchmark.py:81-84), so the allreduce averages genuinely different gradients
        if data_seed_offset is None:
            data_seed_offset = dist.rank()
        self.data, self.target = fixed_synthetic_batch(batch_size, size, self.num_classes, self.device,
                                                       seed=seed + 17 + 1000 * int(data_seed_offset))
        self.batch_size = batch_size
        self.last_loss: Optional[torch.Tensor] = None
        self.steps_done = 0
        self._graph = None

    def loss_fn(self, output, target):
        return ops.aux_classification_loss(output, target, self.num_classes,
                                           getattr(self.model, "aux_loss_weight", None))

    # ---- CUDA-graph replay of the whole step (launch-bound regimes: small per-GPU batches) -------------------------
    def enable_graph(self, warmup: int = 3) -> bool:
        """Capture one full training step (forward, loss, backward with its side-stream weight gradients, the
        per-bucket fused allreduce+SGD kernels) into a CUDA graph and replay it from then on (``graph_step.py``).
        Returns False (and stays eager) when the step cannot be captured: CPU, no fused engine, NVTX profiling."""
        from .graph_step import GraphedStep

        if self._graph is not None:
            return True
        if not self.cuda or self.profile or not GraphedStep.applicable(self.model, self.optimizer, self.data):
            return False
        g = GraphedStep(self._eager_step, self.optimizer, log)
        if not g.capture((self.data, self.target), warmup):
            return False
        self._graph = g
        return True

    def step(self, data=None, target=None):
        data = self.data if data is None else data
        target = self.target if target is None else target
        maybe_inject(self.steps_done, dist.rank())
        self.steps_done += 1
        if self._graph is not None:
            self.last_loss = self._graph(data, target)
            return self.last_loss
        return self._eager_step(data, target)

    def _eager_step(self, data, target):
        if self.profile:        # NVTX ranges: forward / backward (+ overlapped bucket kernels) / step join
            nvtx = torch.cuda.nvtx
            self.optimizer.zero_grad()
            nvtx.range_push("forward")
            output = self.model(data)
            loss = self.loss_fn(output, target)
            nvtx.range_pop()
            nvtx.range_push("backward+allreduce")
            loss.backward()
            nvtx.range_pop()
            nvtx.range_push("optimizer.step(join)")
            self.optimizer.step()
            nvtx.range_pop()
        else:
            self.optimizer.zero_grad()
            output = self.model(data)
            loss = self.loss_fn(output, target)
            loss.backward()
            self.optimizer.step()
        self.last_loss = loss.detach()
        return self.last_loss

    def sync(self):
        if self.cuda:
            torch.cuda.synchronize()


def phase_times(session: BenchmarkSession, steps: int = 5) -> Dict[str, float]:
    """Device time (CUDA events, ms/step, max over ranks) of the phases of an EAGER step: forward + loss, backward (with
    the bucket kernels it overlaps), the optimizer join, and the sum of the bucket kernels' own durations."""
    if not session.cuda:
        return {}
    opt = session.optimizer
    ev = lambda: torch.cuda.Event(enable_timing=True)
    graph, session._graph = session._graph, None
    bucket_ms = []
    if hasattr(opt, "use_python_hooks"):
        opt.use_python_hooks()           # a Python frame per bucket launch is what gets timed here
    orig = getattr(opt, "_launch_bucket", None)
    if orig is not None:
        def timed(b):
            st = opt._comm_stream or torch.cuda.current_stream()
            cur = torch.cuda.current_stream()
            if opt._comm_stream is not None:
                r = ev(); r.record(cur); st.wait_event(r)
            e0, e1 = ev(), ev()
            e0.record(st)
            orig(b)
            e1.record(st)
            bucket_ms.append((e0, e1))
        opt._launch_bucket = timed
    tot = {"forward": 0.0, "backward": 0.0, "step_join": 0.0, "bucket_kernels": 0.0}
    try:
        for _ in range(steps):
            bucket_ms.clear()
            a, b, c, d = ev(), ev(), ev(), ev()
            a.record()
            opt.zero_grad()
            out = session.model(session.data)
            loss = session.loss_fn(out, session.target)
            b.record()
            loss.backward()
            c.record()
            opt.step()
            d.record()
            torch.cuda.synchronize()
            tot["forward"] += a.elapsed_time(b)
            tot["backward"] += b.elapsed_time(c)
            tot["step_join"] += c.elapsed_time(d)
            tot["bucket_kernels"] += sum(x.elapsed_time(y) for x, y in bucket_ms)
    finally:
        if orig is not None:
            opt._launch_bucket = orig
        session._graph = graph
    return {k: dist.allreduce_scalar(v / steps, op="max") for k, v in tot.items()}


def timed_steps(session: BenchmarkSession, n: int) -> float:
    """Milliseconds for ``n`` steps: CUDA events on the launching stream (CPU: perf_counter), max over ranks."""
    import time

    if session.cuda:
        start, stop = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        torch.cuda.synchronize()
        start.record()
        for _ in range(n):
            session.step()
        stop.record()
        stop.synchronize()
        ms = start.elapsed_time(stop)
    else:
        t0 = time.perf_counter()
        for _ in range(n):
            session.step()
        ms = (time.perf_counter() - t0) * 1e3
    return dist.allreduce_scalar(ms, op="max")


def run(args) -> Dict:
    cuda = (not args.no_cuda) and torch.cuda.is_available()
    if args.no_cuda:
        import os

        os.environ["DDL_NO_CUDA"] = "1"
    dist.init()
    if getattr(args, "precision", "bf16") == "fp8":
        if not cuda:
            raise SystemExit("--precision fp8 needs a CUDA device")
        from ..ops import fp8

        fp8.enable(True)
    session = BenchmarkSession(args.model, args.batch_size, cuda, args.fp16_allreduce, args.lr, args.momentum,
                               profile=args.profile)
    device = "GPU" if cuda else "CPU"
    log("Model: %s" % args.model)
    log("Batch size: %d" % args.batch_size)
    log("Number of %ss: %d" % (device, dist.size()))
    log("Running warmup...")
    timed_steps(session, args.num_warmup_batches)
    if getattr(args, "cuda_graph", False) and cuda:
        log("CUDA graph: %s" % ("captured" if session.enable_graph() else "not applicable, running eager"))
    log("Running benchmark...")
    img_secs: List[float] = []
    for x in range(args.num_iters):
        ms = timed_steps(session, args.num_batches_per_iter)
        img_sec = args.batch_size * args.num_batches_per_iter / (ms / 1e3)
        log("Iter #%d: %.1f img/sec per %s" % (x, img_sec, device))
        img_secs.append(img_sec)
    if hasattr(session.optimizer, "check_errors"):
        session.optimizer.check_errors()
    phases = phase_times(session) if getattr(args, "phase_times", False) else {}
    if phases:
        log("Phase ms/step (eager, device-timed): " + ", ".join(f"{k} {v:.3f}" for k, v in phases.items()))
    mean, conf = float(np.mean(img_secs)), float(1.96 * np.std(img_secs))
    log("Img/sec per %s: %.1f +-%.1f" % (device, mean, conf))
    log("Total img/sec on %d %s(s): %.1f +-%.1f" % (dist.size(), device, dist.size() * mean, dist.size() * conf))
    result = {"model": args.model, "batch_size": args.batch_size, "world_size": dist.size(), "device": device,
              "img_sec_per_device": mean, "img_sec_conf": conf, "total_img_sec": dist.size() * mean,
              "iters": img_secs, "phase_ms": phases, "final_loss": float(session.last_loss) if session.last_loss is not None else None}
    if args.json and dist.rank() == 0:
        if args.json == "-":
            print(json.dumps(result))
        else:
            with open(args.json, "w") as f:
                json.dump(result, f)
    return result


def main(argv=None) -> int:
    args = build_parser().parse_args(argv)
    try:
        run(args)
    finally:
        dist.shutdown()
    return 0


if __name__ == "__main__":
    sys.exit(main())
