"""Sharded record files: the TFRecord path of the reference collapsed onto a torch-native format.

Parity: reference ``scripts/convert_imagenet_to_tf_records.py`` (find image files with a seed-42
shuffle ``:418-490``; 1014 train / 128 validation shards ``:507-529``; skip-on-decode-error
``:328-333``; PNG/CMYK normalisation to RGB JPEG ``:149-184``) and the TF readers that shard FILES
across ranks (``data/tfrecords.py:136-141``, ``dataset.shard(hvd.size(), hvd.rank())``).

Format (one file per shard, ``<split>-%05d-of-%05d.rec``): a sequence of
``[u32 label][u32 nbytes][nbytes of JPEG]`` records, little endian.  ``RecordDataset`` gives rank
r the shards r, r+size, ... — the same file-level sharding as the reference's TF input functions.
"""
from __future__ import annotations

import io
import os
import random
import struct
from typing import Iterator, List, Optional, Tuple

import torch

_HDR = struct.Struct("<II")


def find_image_files(root: str, seed: int = 42) -> Tuple[List[str], List[int], List[str]]:
    classes = sorted(d for d in os.listdir(root) if os.path.isdir(os.path.join(root, d)))
    files, labels = [], []
    for i, c in enumerate(classes):
        for f in sorted(os.listdir(os.path.join(root, c))):
            if f.lower().endswith((".jpeg", ".jpg", ".png")):
                files.append(os.path.join(root, c, f))
                labels.append(i)
    order = list(range(len(files)))
    random.Random(seed).shuffle(order)
    return [files[i] for i in order], [labels[i] for i in order], classes


def _as_rgb_jpeg(path: str) -> Optional[bytes]:
    with open(path, "rb") as f:
        raw = f.read()
    try:
        from PIL import Image

        img = Image.open(io.BytesIO(raw))
        if img.format == "JPEG" and img.mode == "RGB":
            return raw
        buf = io.BytesIO()
        img.convert("RGB").save(buf, format="JPEG", quality=100)
        return buf.getvalue()
    except Exception:
        return None          # reference behaviour: skip undecodable files


def write_shards(files: List[str], labels: List[int], out_dir: str, split: str, num_shards: int) -> int:
    os.makedirs(out_dir, exist_ok=True)
    num_shards = max(1, min(num_shards, max(len(files), 1)))
    written = 0
    for s in range(num_shards):
        lo, hi = len(files) * s // num_shards, len(files) * (s + 1) // num_shards
        path = os.path.join(out_dir, f"{split}-{s:05d}-of-{num_shards:05d}.rec")
        with open(path + ".tmp", "wb") as f:
            for p, y in zip(files[lo:hi], labels[lo:hi]):
                data = _as_rgb_jpeg(p)
                if data is None:
                    continue
                f.write(_HDR.pack(y, len(data)))
                f.write(data)
                written += 1
        os.replace(path + ".tmp", path)
    return written


def convert(data_dir: str, out_dir: str, shards_train: int = 1014, shards_val: int = 128) -> dict:
    out = {}
    for split, sub, n in (("train", "train", shards_train), ("validation", "validation", shards_val)):
        root = os.path.join(data_dir, sub)
        if not os.path.isdir(root):
            continue
        files, labels, _ = find_image_files(root)
        out[split] = write_shards(files, labels, os.path.join(out_dir, sub), split, n)
    print(out)
    return out


class RecordDataset(torch.utils.data.IterableDataset):
    """Streams (image tensor, label) from this rank's shards; optional transform on the PIL image."""

    def __init__(self, directory: str, split: str, rank: int = 0, world: int = 1, transform=None, shuffle_seed=None):
        self.files = sorted(os.path.join(directory, f) for f in os.listdir(directory)
                            if f.startswith(split + "-") and f.endswith(".rec"))
        self.files = self.files[rank::world]
        self.transform, self.seed = transform, shuffle_seed

    def __iter__(self) -> Iterator[Tuple[torch.Tensor, int]]:
        from PIL import Image

        info = torch.utils.data.get_worker_info()
        files = self.files if info is None else self.files[info.id::info.num_workers]
        if self.seed is not None:
            files = list(files)
            random.Random(self.seed).shuffle(files)
        for path in files:
            with open(path, "rb") as f:
                while True:
                    hdr = f.read(_HDR.size)
                    if len(hdr) < _HDR.size:
                        break
                    y, n = _HDR.unpack(hdr)
                    img = Image.open(io.BytesIO(f.read(n))).convert("RGB")
                    yield (self.transform(img) if self.transform else img), y


def count_records(path: str) -> int:
    """Number of records in one shard (header walk with seeks: no image bytes are read)."""
    n = 0
    size = os.path.getsize(path)
    with open(path, "rb") as f:
        pos = 0
        while pos + _HDR.size <= size:
            f.seek(pos)
            _, nbytes = _HDR.unpack(f.read(_HDR.size))
            pos += _HDR.size + nbytes
            n += 1
    return n


class RecordLoader:
    """Batched loader over THIS rank's record shards — the trainer-facing end of the record path.

    Parity: the reference's TF input functions give every rank a disjoint subset of the shard FILES
    (``TensorFlow_imagenet/src/data/tfrecords.py:130-141``: ``dataset.shard(hvd.size(), hvd.rank())`` on the file list,
    shuffled per epoch) and its tasks select them with ``--data_type tfrecords``
    (``TensorFlow_imagenet/tensorflow_imagenet.py:110-151``).  Here ``RecordDataset`` does the file-level sharding
    (rank r reads shards r, r+size, ...; DataLoader workers split those again), ``set_epoch`` reseeds the shard order,
    and ``len()`` is the number of batches EVERY rank runs (the minimum over ranks, so collectives stay in step).
    ``augment``: ``host`` or ``device`` (``data/images.py``).
    """

    def __init__(self, directory: str, split: str, batch_size: int, train: bool, size: int = 224, num_workers: int = 4,
                 rank: int = 0, world: int = 1, normalize_on_host: bool = True, seed: int = 0, augment: str = "host"):
        from .images import worker_transform

        transform, collate = worker_transform(train, size, augment, normalize_on_host)
        self.dataset = RecordDataset(directory, split, rank, world, transform, shuffle_seed=seed if train else None)
        all_files = sorted(os.path.join(directory, f) for f in os.listdir(directory)
                           if f.startswith(split + "-") and f.endswith(".rec"))
        if not all_files:
            raise FileNotFoundError(f"no {split}-*.rec shards in {directory}")
        counts = [count_records(p) for p in all_files]
        self.total = sum(counts)
        per_rank = [sum(counts[r::world]) for r in range(world)]
        self.per_rank = min(per_rank)                           # samples every rank is guaranteed to have
        self.batch_size, self.train, self._seed = batch_size, train, seed
        workers = min(num_workers, max(1, len(self.dataset.files)))
        self._loader = torch.utils.data.DataLoader(self.dataset, batch_size=batch_size, num_workers=workers,
                                                   pin_memory=torch.cuda.is_available(), drop_last=False,
                                                   collate_fn=collate)
        self._batches = -(-self.per_rank // batch_size) if self.per_rank else 0

    def set_epoch(self, epoch: int) -> None:
        if self.train:
            self.dataset.seed = self._seed + epoch

    def __len__(self) -> int:
        return self._batches

    def __iter__(self):
        for i, batch in enumerate(self._loader):
            if i >= self._batches:
                break                                            # ranks with more samples stop with the others
            yield batch
