#!/usr/bin/env python
"""Multi-GPU validation + bandwidth sweep of the hand-written NVLink kernels (run under torchrun).

1. correctness: FusedSGD (allreduce + average + SGD + bf16 refresh + grad clear in one kernel per bucket)
   vs the same maths done with torch ops on the gathered per-rank gradients — fp32 wire and bf16 wire,
   multicast (NVLS) and peer-to-peer transports; replicas must stay bit-identical; broadcast kernel.
2. sweep: in-place allreduce 64 KiB .. 1 GiB (fp32 / bf16; one-shot / two-shot; NVLS / P2P), device-timed
   with CUDA events, max over ranks, busbw = algbw * 2(N-1)/N, next to NCCL's all_reduce on the same sizes.
With COMM_JSON=PATH the sweep is also written there as JSON.
"""
import json
import os
import sys

import torch
import torch.distributed as td

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from distributeddeeplearning_b200 import _ext  # noqa: E402
from distributeddeeplearning_b200.parallel import Compression, dist  # noqa: E402
from distributeddeeplearning_b200.parallel import selfcheck  # noqa: E402
from distributeddeeplearning_b200.parallel.engine import SymmetricArena  # noqa: E402


def log(*a):
    if dist.rank() == 0:
        print(*a, flush=True)


def check_engine(use_mc, wire, skew_ns=0):
    ok, used_mc, _ = selfcheck.check_engine(use_mc, wire, skew_ns=skew_ns, log=log)
    return ok, used_mc


def sweep(max_bytes):
    C = _ext.load()
    world, rank = dist.size(), dist.rank()
    dev = torch.device("cuda", torch.cuda.current_device())
    arena = SymmetricArena([("flags", int(C.SIGNAL_PAD_BYTES)), ("data", 2 * max_bytes)], dev, None)
    epochs = torch.zeros(int(C.COMM_CHANNELS) * int(C.MAX_COMM_BLOCKS), dtype=torch.int32, device=dev)
    err = torch.zeros(1, dtype=torch.int32, device=dev)
    off = arena.offsets
    ctx = C.CommCtx(arena.peer_ptrs, arena.mc_ptr, rank, world, off["flags"], 0, 0, 0, 0, epochs.data_ptr(),
                    err.data_ptr(), int(30e9))
    st = torch.cuda.current_stream().cuda_stream
    results = []
    sizes = [1 << k for k in range(16, 31) if (1 << k) <= max_bytes]
    # correctness of the plain allreduce first
    n = 1 << 20
    for bf16 in (False, True):
        for use_mc in ([True, False] if arena.has_multicast else [False]):
            for oneshot in (False, True):
                dt = torch.bfloat16 if bf16 else torch.float32
                buf = arena.region("data", dt, 2 * n)
                buf[:n] = (torch.arange(n, device=dev) % 13).to(dt) * (rank + 1)
                torch.cuda.synchronize()
                td.barrier()
                C.allreduce(ctx, 4, off["data"], n, bf16, 1.0, use_mc, oneshot, 32, st)
                torch.cuda.synchronize()
                out = buf[n:2 * n] if oneshot else buf[:n]
                exp = (torch.arange(n, device=dev) % 13).float() * (world * (world + 1) / 2)
                good = bool(torch.allclose(out.float(), exp, rtol=1e-2 if bf16 else 1e-6))
                log(f"[{'ok' if good else 'FAIL'}] allreduce {'bf16' if bf16 else 'fp32'} {'nvls' if use_mc else 'p2p'} "
                    f"{'one-shot' if oneshot else 'two-shot'}")
                td.barrier()
    for nbytes in sizes:
        for bf16 in (False, True):
            es = 2 if bf16 else 4
            numel = nbytes // es
            variants = []
            if arena.has_multicast:
                variants += [("nvls-2shot", True, False)]
                if nbytes <= (8 << 20):
                    variants += [("nvls-1shot", True, True)]
            variants += [("p2p-2shot", False, False)]
            if nbytes <= (8 << 20):
                variants += [("p2p-1shot", False, True)]
            for blocks in (16, 32, 64):
                for name, use_mc, oneshot in variants:
                    def run():
                        C.allreduce(ctx, 4, off["data"], numel, bf16, 1.0, use_mc, oneshot, blocks, st)
                    for _ in range(3):
                        run()
                    torch.cuda.synchronize()
                    td.barrier()
                    a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
                    reps = 20 if nbytes <= (16 << 20) else 5
                    a.record()
                    for _ in range(reps):
                        run()
                    b.record()
                    b.synchronize()
                    ms = dist.allreduce_scalar(a.elapsed_time(b) / reps, op="max")
                    algbw = nbytes / ms / 1e6
                    results.append({"bytes": nbytes, "dtype": "bf16" if bf16 else "fp32", "impl": name, "blocks": blocks,
                                    "ms": ms, "algbw_gbs": algbw, "busbw_gbs": algbw * 2 * (world - 1) / world})
            # NCCL reference on the same size
            t = torch.zeros(numel, dtype=torch.bfloat16 if bf16 else torch.float32, device=dev)
            for _ in range(3):
                td.all_reduce(t)
            torch.cuda.synchronize()
            td.barrier()
            a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            reps = 20 if nbytes <= (16 << 20) else 5
            a.record()
            for _ in range(reps):
                td.all_reduce(t)
            b.record()
            b.synchronize()
            ms = dist.allreduce_scalar(a.elapsed_time(b) / reps, op="max")
            algbw = nbytes / ms / 1e6
            results.append({"bytes": nbytes, "dtype": "bf16" if bf16 else "fp32", "impl": "nccl", "blocks": 0, "ms": ms,
                            "algbw_gbs": algbw, "busbw_gbs": algbw * 2 * (world - 1) / world})
        best = {}
        for r in results:
            if r["bytes"] == nbytes and r["dtype"] == "fp32":
                k = r["impl"]
                if k not in best or r["ms"] < best[k]["ms"]:
                    best[k] = r
        log(f"{nbytes >> 10:>8d} KiB fp32: " + "  ".join(f"{k} {v['ms'] * 1e3:8.1f}us {v['busbw_gbs']:6.1f}GB/s(b{v['blocks']})"
                                                        for k, v in sorted(best.items())))
    if int(err.item()):
        log("barrier timeout flag set:", int(err.item()))
    return results


def main():
    dist.init()
    world = dist.size()
    log(f"world={world} device={torch.cuda.get_device_name()}")
    oks = []
    ok, had_mc = check_engine(None, Compression.none)
    oks.append(ok)
    oks.append(check_engine(None, Compression.bf16)[0])
    if had_mc:
        oks.append(check_engine(False, Compression.none)[0])
        oks.append(check_engine(False, Compression.bf16)[0])
    # de-synchronised blocks / ranks: a producer-consumer block mismatch in the protocol shows up as wrong sums here
    for wire in (Compression.none, Compression.bf16):
        oks.append(check_engine(None, wire, skew_ns=30000)[0])
        if had_mc:
            oks.append(check_engine(False, wire, skew_ns=30000)[0])
    if "--model-check" in sys.argv:
        eq = selfcheck.step_equivalence("resnet50", 32)
        log("STEP EQUIVALENCE:", json.dumps(eq))
        oks.append(eq["ok"])
    max_bytes = int(os.environ.get("SWEEP_MAX", 1 << 30))
    res = [] if "--no-sweep" in sys.argv else sweep(max_bytes)
    if dist.rank() == 0 and res and os.environ.get("COMM_JSON"):
        json.dump({"world": world, "multicast": had_mc, "results": res, "engine_checks_ok": all(oks)},
                  open(os.environ["COMM_JSON"], "w"), indent=1)
    log("ENGINE CHECKS:", "all ok" if all(oks) else "FAILURES")
    dist.shutdown()
    return 0 if all(oks) else 1


if __name__ == "__main__":
    sys.exit(main())
