#!/usr/bin/env python
"""Per-bucket timeline of the fused allreduce+SGD kernels inside a real training step (run under torchrun).

For each gradient bucket of ResNet-50 (or --model) at batch --batch-size, in EAGER mode (so CUDA events can be placed
between the launches): when the bucket became ready relative to the start of backward, how long its kernel ran on the
comm stream (barrier-in wait + data phase [+ closing barrier on the last bucket]), and how much of the step was exposed
after the last weight-gradient kernel (= what data parallelism costs on top of the single-GPU step).  Also reports the
achieved fraction of the per-bucket roofline S*(1 + 1/N) bytes / 450 GB/s (NVLink 4 per direction on H100; NVLS two-shot: each rank pulls its
1/N slice through the switch and pushes S/N fp32 weights + S/N/2 bf16 copies + S/N zeros to every replica).
Max over ranks per bucket; --json PATH also writes the timeline as JSON.
"""
import argparse
import json
import os
import sys

import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from distributeddeeplearning_b200.parallel import dist  # noqa: E402
from distributeddeeplearning_b200.workloads.benchmark import BenchmarkSession  # noqa: E402


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--model", default="resnet50")
    ap.add_argument("--batch-size", type=int, default=256)
    ap.add_argument("--steps", type=int, default=6)
    ap.add_argument("--fp16-allreduce", action="store_true")
    ap.add_argument("--json", default=None)
    a = ap.parse_args()
    dist.init()
    rank, world = dist.rank(), dist.size()
    s = BenchmarkSession(a.model, a.batch_size, True, a.fp16_allreduce, data_seed_offset=rank)
    opt = s.optimizer
    for _ in range(4):
        s.step()
    torch.cuda.synchronize()
    nb = opt.num_buckets
    rec = []
    opt.use_python_hooks()              # the timeline wraps the Python bucket launch
    orig = opt._launch_bucket

    def timed_launch(b):
        cur = torch.cuda.current_stream()
        ready = torch.cuda.Event(enable_timing=True)
        ready.record(cur)                                   # the bucket's last gradient hook fired here (main stream)
        st = opt._comm_stream or cur
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        # start event AFTER the comm stream has waited for readiness: kernel time, not the wait for backward
        if opt._comm_stream is not None:
            st.wait_event(ready)
        from distributeddeeplearning_b200.ops.functional import wgrad_join
        wgrad_join(st)
        e0.record(st)
        orig(b)
        e1.record(st)
        rec[-1]["buckets"].append((b, ready, e0, e1))

    opt._launch_bucket = timed_launch
    out_steps = []
    for _ in range(a.steps):
        rec.append({"buckets": []})
        t0, t_bwd, t_end = (torch.cuda.Event(enable_timing=True) for _ in range(3))
        t0.record()
        opt.zero_grad()
        out = s.model(s.data)
        loss = s.loss_fn(out, s.target)
        loss.backward()
        t_bwd.record()                                       # main stream: all dgrad/wgrad launches enqueued
        opt.step()
        t_end.record()
        torch.cuda.synchronize()
        st = {"step_ms": t0.elapsed_time(t_end), "fwd_bwd_ms": t0.elapsed_time(t_bwd),
              "exposed_after_backward_ms": t_bwd.elapsed_time(t_end), "buckets": []}
        for (b, ready, e0, e1) in rec[-1]["buckets"]:
            numel = int(opt.plan["bucket_numel"][b])
            st["buckets"].append({"bucket": b, "mbytes": numel * 4 / 1e6, "ready_at_ms": t0.elapsed_time(ready),
                                  "start_at_ms": t0.elapsed_time(e0), "kernel_ms": e0.elapsed_time(e1),
                                  "end_at_ms": t0.elapsed_time(e1)})
        out_steps.append(st)
    last = out_steps[-1]
    # max over ranks
    for bk in last["buckets"]:
        bk["kernel_ms"] = dist.allreduce_scalar(bk["kernel_ms"], op="max")
    for k in ("step_ms", "fwd_bwd_ms", "exposed_after_backward_ms"):
        last[k] = dist.allreduce_scalar(last[k], op="max")
    if rank == 0:
        wire = 2 if a.fp16_allreduce else 4
        print(f"model={a.model} batch={a.batch_size} world={world} engine={opt.describe()}")
        print(f"step {last['step_ms']:.3f} ms (eager), fwd+bwd enqueue span {last['fwd_bwd_ms']:.3f} ms, "
              f"exposed after backward {last['exposed_after_backward_ms']:.3f} ms")
        print("| bucket | MB (fp32) | ready at ms | kernel start | kernel ms | roofline ms | achieved |")
        print("|---|---|---|---|---|---|---|")
        for bk in last["buckets"]:
            S = bk["mbytes"] * 1e6
            # NVLS two-shot wire per GPU: the reduce phase delivers this rank's S/N slice, the broadcast phase pushes
            # S/N of results to the switch and every replica receives S: ~S * (1 + 1/N) bytes at 450 GB/s per direction (NVLink 4)
            Sw = S * wire / 4
            roof = Sw * (1.0 + 1.0 / world) / 450e9 * 1e3 if world > 1 else 0.0
            bk["roofline_ms"] = roof
            bk["achieved"] = roof / bk["kernel_ms"] if bk["kernel_ms"] > 0 else 0
            print(f"| {bk['bucket']} | {bk['mbytes']:.2f} | {bk['ready_at_ms']:.2f} | {bk['start_at_ms']:.2f} | "
                  f"{bk['kernel_ms']:.3f} | {roof:.3f} | {bk['achieved']:.2f} |")
        if a.json:
            json.dump({"world": world, "model": a.model, "batch": a.batch_size, "steps": out_steps}, open(a.json, "w"),
                      indent=1)
    dist.shutdown()


if __name__ == "__main__":
    main()
