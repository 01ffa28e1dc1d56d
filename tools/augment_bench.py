#!/usr/bin/env python
"""Device augmentation (augment="device") against the host PIL path on a seeded JPEG folder with an ImageNet-like size
spread:

1. ``resized_crop`` kernel time at batch 256 for train and validation descriptors (CUDA events over many launches), with
   bytes read / written from the descriptors and GB/s, against torchvision v2 ``resized_crop`` + ``normalize`` on CUDA
   uint8 tensors, one image at a time;
2. steady-state loader throughput (img/s, through the copy and the device step) of both paths at several
   ``num_workers`` up to ``os.cpu_count()``: the first 2 x num_workers batches (the DataLoader's prefetch) are not
   timed, then at least 10 batches per worker are; the runs alternate and the whole set runs twice;
3. the ImageNet trainer's img/s on resnet50 for both paths (the second epoch of two).

Stages 2 and 3 read the folder ``--copies`` times over (symbolic links), so their windows hold many batches per
worker without generating more JPEGs.

Prints the card name and power limit.  ``--quick`` shrinks every stage (a check that the tool runs).
"""
import argparse
import json
import os
import re
import subprocess
import sys
import tempfile
import time

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(HERE)
sys.path.insert(0, ROOT)


def _write_image(args):
    import numpy as np
    from PIL import Image

    path, seed = args
    rng = np.random.default_rng(seed)
    u = rng.random()
    short = int(rng.integers(333, 501)) if u < 0.85 else (int(rng.integers(800, 1501)) if u < 0.95
                                                           else int(rng.integers(80, 224)))
    ar = (4 / 3, 3 / 4, 1.0)[int(rng.integers(0, 3))]
    w, h = (int(short * ar), short) if ar >= 1 else (short, int(short / ar))
    y, x = np.mgrid[0:h, 0:w].astype(np.float32)
    f = rng.uniform(5, 40, 3)
    a = 127 + 60 * np.sin(x[..., None] / f) + 50 * np.cos(y[..., None] / f[::-1])
    a += rng.integers(-40, 41, (h, w, 3), dtype=np.int8)
    Image.fromarray(np.clip(a, 0, 255).astype(np.uint8)).save(path, quality=90)


def make_folder(root, n, classes=4, seed=0):
    """``n`` seeded JPEGs (quality 90) in ``classes`` class folders, written in parallel (each image from its own
    seed).  Sizes follow ImageNet's spread: mostly a shorter side of 333-500 at 4:3, 3:4 or 1:1, one in ten 800-1500,
    one in twenty smaller than 224."""
    from concurrent.futures import ProcessPoolExecutor

    for c in range(classes):
        os.makedirs(os.path.join(root, f"n{c:08d}"), exist_ok=True)
    jobs = [(os.path.join(root, f"n{k % classes:08d}", f"img{k:06d}.jpg"), seed * 1_000_003 + k) for k in range(n)]
    with ProcessPoolExecutor(max_workers=min(16, os.cpu_count() or 1)) as ex:
        list(ex.map(_write_image, jobs, chunksize=16))
    return root


def expand_folder(src, dst, copies):
    """``dst``: the class folders of ``src`` with every image linked ``copies`` times (distinct file names)."""
    for c in sorted(os.listdir(src)):
        os.makedirs(os.path.join(dst, c), exist_ok=True)
        for f in sorted(os.listdir(os.path.join(src, c))):
            for k in range(copies):
                os.symlink(os.path.join(src, c, f), os.path.join(dst, c, f"{k}_{f}"))
    return dst


def card():
    import torch

    r = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                       capture_output=True, text=True)
    return r.stdout.strip().splitlines()[0] if r.returncode == 0 and r.stdout.strip() else torch.cuda.get_device_name()


def packed_batch(root, train, size, n, seed=0):
    """One collated device-path batch of the first ``n`` images of the folder (crop boxes drawn from ``seed``)."""
    import torch
    from torchvision import datasets

    from distributeddeeplearning_b200.data import images

    torch.manual_seed(seed)
    ds = datasets.ImageFolder(root, images.DeviceAugmentTransform(train, size))
    return images.collate_regions([ds[i % len(ds)] for i in range(n)])[0]


def bench_kernel(root, size, iters):
    import torch
    from torchvision.transforms.v2 import functional as TF

    from distributeddeeplearning_b200.data import images
    from distributeddeeplearning_b200.ops import native

    dev = torch.device("cuda")
    aug = images.DeviceAugment(dev, size)
    out = {}
    for split, train in (("train", True), ("val", False)):
        batch = packed_batch(root, train, size, 256).pin_memory().to(dev)
        for _ in range(5):
            aug(batch)
        torch.cuda.synchronize()
        a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        a.record()
        for _ in range(iters):
            aug(batch)
        b.record()
        torch.cuda.synchronize()
        us = a.elapsed_time(b) * 1e3 / iters
        d = batch.desc
        read = int((d[:, 1] * d[:, 2] * 3).sum())
        written = 256 * size * size * 8
        # torchvision v2 on the same regions, one image at a time (uint8 CUDA tensors, antialiased bilinear); timed
        # per batch of 256, like the kernel
        regs, params = [], []
        for off, hr, wr, sy, sx, oy, ox, flip in d.tolist():
            off, hr, wr = int(off), int(hr), int(wr)
            regs.append(batch.data[off:off + hr * wr * 3].view(hr, wr, 3).permute(2, 0, 1))
            if train:
                params.append((0, 0, hr, wr, (size, size), None))
            else:
                rh, rw = round(hr / sy), round(wr / sx)
                params.append((int(oy), int(ox), size, size, None, (rh, rw)))
        mean, std = list(images.RGB_MEAN), list(images.RGB_SD)

        def tv():
            for r, (top, left, h, w, tsize, resize) in zip(regs, params):
                if resize is None:
                    x = TF.resized_crop(r, top, left, h, w, list(tsize), antialias=True)
                else:
                    x = TF.crop(TF.resize(r, list(resize), antialias=True), top, left, h, w)
                TF.normalize(TF.to_dtype(x, torch.float32, scale=True), mean, std)
        tv()
        torch.cuda.synchronize()
        a.record()
        reps = max(1, iters // 20)
        for _ in range(reps):
            tv()
        b.record()
        torch.cuda.synchronize()
        tv_us = a.elapsed_time(b) * 1e3 / reps
        out[split] = {"kernel_us": round(us, 1), "bytes_read": read, "bytes_written": written,
                      "GBps": round((read + written) / us / 1e3, 1), "torchvision_v2_batch_us": round(tv_us, 1),
                      "torchvision_v2_per_image_us": round(tv_us / 256, 1),
                      "speedup_vs_torchvision": round(tv_us / us, 1)}
        print(f"kernel {split}: {json.dumps(out[split])}", flush=True)
    return out


def bench_loader(root, size, workers, batch_size):
    import torch

    from distributeddeeplearning_b200.data import images

    dev = torch.device("cuda")
    res = {}

    def run(augment, nw):
        loader, _ = images.image_folder_loader(root, batch_size, True, size, nw, device_normalize=True,
                                               augment=augment)
        prep = images.DeviceAugment(dev, size) if augment == "device" else images.DeviceNormalizer(dev)
        # the DataLoader keeps 2 batches per worker in flight: those fill while the workers start, so they are not
        # timed; the window then holds at least 10 batches per worker
        warm, timed = 2 * nw, max(10 * nw, 16)
        if len(loader) < warm + timed:
            raise SystemExit(f"loader stage needs {(warm + timed) * batch_size} images, the folder has "
                             f"{len(loader.dataset)}: raise --images or --copies")
        it = iter(loader)
        for _ in range(warm):
            x, _ = next(it)
            prep(x.to(dev, non_blocking=True))
        torch.cuda.synchronize()
        n, t0 = 0, time.perf_counter()
        for _ in range(timed):
            x, y = next(it)
            prep(x.to(dev, non_blocking=True))
            n += len(y)
        torch.cuda.synchronize()
        dt = time.perf_counter() - t0
        del it, loader
        return n / dt

    for rep in range(2):
        for nw in workers:
            for augment in (("host", "device") if rep == 0 else ("device", "host")):
                v = run(augment, nw)
                res.setdefault(f"{augment}@{nw}", []).append(round(v, 1))
                print(f"loader run {rep} workers {nw} {augment}: {v:.1f} img/s", flush=True)
    return res


def bench_trainer(root, batch_size, workers):
    out = {}
    for augment in ("host", "device"):
        with tempfile.TemporaryDirectory() as tmp:
            env = dict(os.environ, PYTHONPATH=ROOT, DDL_LOG_DIR=os.path.join(tmp, "logs"), DDL_RUN_DIR=tmp)
            r = subprocess.run([sys.executable, "-m", "distributeddeeplearning_b200.workloads.imagenet", "--epochs", "2",
                                "--batch_size", str(batch_size), "--use_gpu", "True", "--training_data_path", root,
                                "--num_workers", str(workers), "--augment", augment, "--model", "resnet50"],
                               cwd=tmp, env=env, capture_output=True, text=True, timeout=3600)
        log = r.stdout + r.stderr
        took = re.findall(r"Training epoch (\d+) took ([\d.]+)", log)
        if r.returncode != 0 or len(took) < 2:
            print(log[-3000:], flush=True)
            raise SystemExit(f"trainer ({augment}) failed")
        n = sum(len(fs) for _, _, fs in os.walk(root))
        out[augment] = {"epoch2_seconds": float(took[1][1]), "img_per_s": round(n / float(took[1][1]), 1),
                        "graph_captured": "captured into a CUDA graph" in log}
        print(f"trainer resnet50 {augment}: {json.dumps(out[augment])}", flush=True)
    return out


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--images", type=int, default=3072)
    ap.add_argument("--size", type=int, default=224)
    ap.add_argument("--iters", type=int, default=200)
    ap.add_argument("--batch-size", type=int, default=256)
    ap.add_argument("--loader-batch-size", type=int, default=64)
    ap.add_argument("--copies", type=int, default=4, help="times the loader and trainer stages read each image")
    ap.add_argument("--workers", default=None, help="comma-separated worker counts (default 1, 2, 4, ... cpu_count)")
    ap.add_argument("--trainer-workers", type=int, default=None)
    ap.add_argument("--stages", default="kernel,loader,trainer", help="comma-separated subset of kernel,loader,trainer")
    ap.add_argument("--quick", action="store_true")
    ap.add_argument("--out", default=None, help="write the results as JSON here")
    a = ap.parse_args()
    import torch

    if not torch.cuda.is_available():
        raise SystemExit("augment_bench needs a GPU")
    if a.quick:
        a.images, a.iters, a.batch_size, a.loader_batch_size, a.copies = 256, 20, 64, 4, 1
        a.workers = a.workers or "1,2"
    cpus = os.cpu_count() or 1
    if a.workers:
        workers = [int(w) for w in a.workers.split(",")]
    else:
        workers = sorted({min(w, cpus) for w in (1, 2, 4, 8, 16, 32, 64, cpus)})
    print(f"card: {card()}  cpu_count: {cpus}", flush=True)
    res = {"card": card(), "cpu_count": cpus}
    with tempfile.TemporaryDirectory() as tmp:
        root = make_folder(os.path.join(tmp, "train"), a.images)
        many = expand_folder(root, os.path.join(tmp, "train_x%d" % a.copies), a.copies)
        stages = a.stages.split(",")
        if "kernel" in stages:
            res["kernel"] = bench_kernel(root, a.size, a.iters)
        if "loader" in stages:
            res["loader_batch_size"] = a.loader_batch_size
            res["loader"] = bench_loader(many, a.size, workers, a.loader_batch_size)
        if "trainer" in stages:
            res["trainer"] = bench_trainer(many, a.batch_size, a.trainer_workers or cpus)
    print(json.dumps(res), flush=True)
    if a.out:
        os.makedirs(os.path.dirname(os.path.abspath(a.out)), exist_ok=True)
        with open(a.out, "w") as f:
            json.dump(res, f, indent=1)


if __name__ == "__main__":
    main()
