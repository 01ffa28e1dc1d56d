"""Real-image (ImageFolder) pipeline (SURVEY.md K21).

Parity: train = RandomResizedCrop(224) -> RandomHorizontalFlip -> ToTensor -> Normalize,
val = Resize(256) -> CenterCrop(224) -> ToTensor -> Normalize, ``num_workers`` DataLoader workers with
pinned memory (``imagenet_pytorch_horovod.py:336-375``; ``PyTorch_hvd/...:82-111``).

Two augmentation paths:

* ``augment="host"`` (default; the reference's PIL pipeline pixel for pixel, and the only path on CPU): the workers
  decode, crop, resize, flip and ``ToTensor``; normalisation + NCHW->NHWC4 + bf16 cast run in ONE device kernel
  (``ops.native.nchw_to_nhwc4``) when ``device_normalize`` is set.
* ``augment="device"``: the workers decode and draw the crop box and flip with the same RNG calls as the host path,
  then ship the uint8 region (``DeviceAugmentTransform``); ``collate_regions`` packs a batch into one buffer plus a
  descriptor per image (``PackedRegions``), and ``DeviceAugment`` resamples, flips and normalises it in one kernel
  (``ops.native.resized_crop``, antialiased bilinear like PIL's ``BILINEAR``).  ``resized_crop_reference`` is its
  float64 twin.
"""
from __future__ import annotations

import numpy as np
import torch

RGB_MEAN = (0.485, 0.456, 0.406)
RGB_SD = (0.229, 0.224, 0.225)


def build_transforms(train: bool, size: int = 224, normalize_on_host: bool = True):
    from torchvision import transforms

    tail = [transforms.ToTensor()]
    if normalize_on_host:
        tail.append(transforms.Normalize(RGB_MEAN, RGB_SD))
    if train:
        return transforms.Compose([transforms.RandomResizedCrop(size), transforms.RandomHorizontalFlip(), *tail])
    return transforms.Compose([transforms.Resize(int(size * 256 / 224)), transforms.CenterCrop(size), *tail])


AUGMENT_PATHS = ("host", "device")


def worker_transform(train: bool, size: int, augment: str, normalize_on_host: bool):
    """(per-sample transform, collate_fn) of one augmentation path."""
    if augment not in AUGMENT_PATHS:
        raise ValueError(f"augment must be host or device, got {augment!r}")
    if augment == "device":
        return DeviceAugmentTransform(train, size), collate_regions
    return build_transforms(train, size, normalize_on_host), None


def image_folder_loader(path: str, batch_size: int, train: bool, size: int = 224, num_workers: int = 5,
                        device_normalize: bool = False, seed: int = 0, augment: str = "host"):
    from torchvision import datasets

    from .sampler import get_sampler

    transform, collate = worker_transform(train, size, augment, normalize_on_host=not device_normalize)
    ds = datasets.ImageFolder(path, transform)
    sampler = get_sampler(ds, shuffle=train)
    loader = torch.utils.data.DataLoader(ds, batch_size=batch_size, sampler=sampler, num_workers=num_workers,
                                         pin_memory=torch.cuda.is_available(), drop_last=False,
                                         persistent_workers=num_workers > 0, collate_fn=collate)
    return loader, sampler


class DeviceNormalizer:
    """(x - mean) / std + layout/dtype conversion in one device pass."""

    def __init__(self, device):
        self.mean = torch.tensor(RGB_MEAN, dtype=torch.float32, device=device)
        self.std = torch.tensor(RGB_SD, dtype=torch.float32, device=device)

    def __call__(self, x: torch.Tensor) -> torch.Tensor:
        from ..ops import native, use_native

        if x.is_cuda and use_native(x):
            return native.nchw_to_nhwc4(x, self.mean, self.std)
        return (x - self.mean.view(1, 3, 1, 1).to(x.device)) / self.std.view(1, 3, 1, 1).to(x.device)


# ------------------------------------------------------------------------------------------------------------------------
# augment="device"
# ------------------------------------------------------------------------------------------------------------------------
class DeviceAugmentTransform:
    """Worker transform of the device path: PIL RGB image -> (uint8 HWC3 region, (Hr, Wr, sy, sx, oy, ox, flip)).

    Train: ``RandomResizedCrop.get_params`` then ``torch.rand(1) < 0.5``, the same calls in the same order as the host
    path's ``Compose``, so a given seed gives every sample the host path's crop box and flip; the region is the crop box
    and the scales are crop / size.  Validation: the region is the whole image, the scales are those of
    ``Resize(int(size * 256 / 224))`` and the offsets are ``CenterCrop(size)``'s top / left."""

    def __init__(self, train: bool, size: int = 224):
        self.train, self.size = train, int(size)

    def __call__(self, img):
        from torchvision import transforms

        S = self.size
        if self.train:
            i, j, h, w = transforms.RandomResizedCrop.get_params(img, (0.08, 1.0), (3.0 / 4.0, 4.0 / 3.0))
            flip = bool(torch.rand(1) < 0.5)
            return np.asarray(img.crop((j, i, j + w, i + h))), (h, w, h / S, w / S, 0, 0, int(flip))
        W, H = img.size
        short = int(S * 256 / 224)
        if W <= H:
            nw, nh = short, int(short * H / W)
        else:
            nh, nw = short, int(short * W / H)
        top, left = int(round((nh - S) / 2.0)), int(round((nw - S) / 2.0))
        return np.asarray(img), (H, W, H / nh, W / nw, top, left, 0)


class PackedRegions:
    """A batch of ragged uint8 HWC3 regions: ``data`` holds them back to back, each at a 16-byte-aligned offset, and
    ``desc`` (float64 [B, 8], always on the host) holds (offset, Hr, Wr, sy, sx, oy, ox, flip) per image.  ``to()``
    moves only ``data``: ``native.resized_crop`` checks the descriptor on the host before it launches."""

    def __init__(self, data: torch.Tensor, desc: torch.Tensor):
        self.data, self.desc = data, desc

    def __len__(self) -> int:
        return int(self.desc.shape[0])

    def pin_memory(self, device=None):
        return PackedRegions(self.data.pin_memory(), self.desc.pin_memory())

    def to(self, device, non_blocking: bool = False):
        return PackedRegions(self.data.to(device, non_blocking=non_blocking), self.desc)


def collate_regions(samples):
    """[((region, (Hr, Wr, sy, sx, oy, ox, flip)), label), ...] -> (PackedRegions, int64 labels)."""
    offsets, total = [], 0
    for (region, _), _ in samples:
        offsets.append(total)
        total += -(-region.size // 16) * 16
    buf = np.empty(max(total, 1), dtype=np.uint8)
    for ((region, _), _), off in zip(samples, offsets):
        buf[off:off + region.size] = region.reshape(-1)
    desc = torch.tensor([[off, *d] for ((_, d), _), off in zip(samples, offsets)], dtype=torch.float64)
    labels = torch.tensor([y for _, y in samples], dtype=torch.int64)
    return PackedRegions(torch.from_numpy(buf), desc), labels


class DeviceAugment:
    """``prepare`` of the device path: a copied ``PackedRegions`` batch -> bf16 NHWC4 [B, size, size] activations."""

    def __init__(self, device, size: int = 224):
        self.size = int(size)
        self.mean = torch.tensor(RGB_MEAN, dtype=torch.float32, device=device)
        self.std = torch.tensor(RGB_SD, dtype=torch.float32, device=device)

    def __call__(self, batch: PackedRegions) -> torch.Tensor:
        from ..ops import native

        return native.resized_crop(batch.data, batch.desc, self.size, self.mean, self.std)


def _axis_weights(L: int, S: int, s: float, o: float) -> torch.Tensor:
    """[S, L] float64 antialiased bilinear (triangle) weights of one axis, taps clamped to [0, L)."""
    center = s * (torch.arange(S, dtype=torch.float64) + o + 0.5)
    support, inv = (s, 1.0 / s) if s >= 1.0 else (1.0, 1.0)
    lo = (center - support + 0.5).trunc().clamp(min=0)
    hi = (center + support + 0.5).trunc().clamp(max=L)
    j = torch.arange(L, dtype=torch.float64)
    w = (1.0 - ((j[None] - center[:, None] + 0.5) * inv).abs()).clamp(min=0)
    w = w * ((j[None] >= lo[:, None]) & (j[None] < hi[:, None]))
    return w / w.sum(1, keepdim=True)


def resized_crop_reference(data: torch.Tensor, desc: torch.Tensor, size: int, mean=None, std=None) -> torch.Tensor:
    """float64 twin of ``native.resized_crop``: [B, 3, size, size] of (v/255 - mean)/std (v/255 without mean / std)."""
    data = data.cpu()
    out = []
    for off, hr, wr, sy, sx, oy, ox, flip in desc.tolist():
        off, hr, wr = int(off), int(hr), int(wr)
        region = data[off:off + hr * wr * 3].view(hr, wr, 3).to(torch.float64)
        wy, wx = _axis_weights(hr, size, sy, oy), _axis_weights(wr, size, sx, ox)
        if flip:
            wx = wx.flip(0)
        rows = (wy @ region.reshape(hr, wr * 3)).view(size, wr, 3)          # vertical pass first: [size, Wr, 3]
        out.append(torch.einsum("ywc,xw->cyx", rows, wx) / 255.0)
    v = torch.stack(out)
    if mean is not None:
        m, s = (torch.tensor(t, dtype=torch.float64).view(1, 3, 1, 1) for t in (mean, std))
        v = (v - m) / s
    return v
