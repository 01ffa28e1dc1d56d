"""CPU tests of the device augmentation path (augment="device", data/images.py + csrc/ops/augment.cu): the float64 twin
of the kernel against torch's antialiased interpolate and against the host PIL pipeline, the device path's crop boxes and
flips against the host path's through both loaders, the collate format, descriptor validation, the trainers' refusals
and the kernel's ptxas figures."""
import os
import re
import shutil
import subprocess

import numpy as np
import pytest
import torch
import torch.nn.functional as F
from PIL import Image

from distributeddeeplearning_b200 import _ext
from distributeddeeplearning_b200.data import images, records
from distributeddeeplearning_b200.ops import native

# PIL resamples with fixed-point weights and stores its horizontal pass as uint8, so it differs from the exact filter by
# up to one uint8 level; ToTensor's float32 v / 255 adds ~1e-5 of a level (observed worst: 1.0000075 levels).
PIL_LEVELS = 1.0 + 1e-4
# the twin against F.interpolate(antialias=True) in float64 (observed worst: 8e-16)
INTERP_TOL = 1e-12


def _photo(w, h, seed):
    """A seeded image with smooth structure and pixel noise (a flat or pure-noise image would hide filter errors)."""
    rng = np.random.default_rng(seed)
    y, x = np.mgrid[0:h, 0:w]
    a = (127 + 60 * np.sin(x / (7.0 + seed % 11)) + 50 * np.cos(y / 23.0))[..., None] + rng.normal(0, 25, (h, w, 3))
    return Image.fromarray(np.clip(a, 0, 255).astype(np.uint8))


# wide, tall, tiny (upscaled at every size), huge, and the ImageNet-typical 500 x 375
SHAPES = [("wide", 800, 200), ("tall", 375, 500), ("tiny", 120, 90), ("huge", 2000, 1500), ("imagenet", 500, 375)]
SIZES = [224, 299, 384, 480, 600]


def _one(img, train, size, seed):
    """(host tensor [3, S, S] in [0, 1], packed device batch of the same sample) with the same RNG state."""
    torch.manual_seed(seed)
    host = images.build_transforms(train, size, normalize_on_host=False)(img)
    torch.manual_seed(seed)
    region, d = images.DeviceAugmentTransform(train, size)(img)
    packed, _ = images.collate_regions([((region, d), 0)])
    return host, packed, region, d


@pytest.mark.parametrize("size", SIZES)
@pytest.mark.parametrize("shape", SHAPES, ids=[s[0] for s in SHAPES])
def test_twin_matches_interpolate_and_pil(shape, size):
    name, w, h = shape
    img = _photo(w, h, seed=size + w)
    for train in (True, False):
        for seed in (0, 1):
            host, packed, region, d = _one(img, train, size, seed)
            twin = images.resized_crop_reference(packed.data, packed.desc, size)[0]
            levels = ((twin - host.double()) * 255).abs().max().item()
            assert levels <= PIL_LEVELS, (name, size, train, seed, levels)
            if train:          # the crop box through torch's antialiased bilinear interpolate, flipped like the host
                reg = torch.from_numpy(np.array(region)).permute(2, 0, 1)[None].double() / 255
                ref = F.interpolate(reg, size=(size, size), mode="bilinear", antialias=True, align_corners=False)[0]
                ref = ref.flip(-1) if d[6] else ref
                assert (ref - twin).abs().max().item() <= INTERP_TOL, (name, size, seed)


def test_twin_normalises_and_flips():
    img = _photo(500, 375, 3)
    region = np.asarray(img)
    packed, _ = images.collate_regions([((region, (375, 500, 375 / 224, 500 / 224, 0, 0, f)), 0) for f in (0, 1)])
    v = images.resized_crop_reference(packed.data, packed.desc, 224)
    assert torch.equal(v[0].flip(-1), v[1])
    n = images.resized_crop_reference(packed.data, packed.desc, 224, images.RGB_MEAN, images.RGB_SD)
    m, s = (torch.tensor(t, dtype=torch.float64).view(3, 1, 1) for t in (images.RGB_MEAN, images.RGB_SD))
    assert torch.allclose(n[0], (v[0] - m) / s, atol=1e-12)


def _folder(root, n_per_class=5):
    sizes = [(500, 375), (375, 500), (120, 90), (800, 200), (640, 480)]
    for c in range(3):
        os.makedirs(os.path.join(root, f"c{c}"), exist_ok=True)
        for k in range(n_per_class):
            w, h = sizes[(c + k) % len(sizes)]
            _photo(w, h, 10 * c + k).save(os.path.join(root, f"c{c}", f"{k}.jpg"), quality=90)
    return root


def _compare(host_batches, dev_batches, size):
    assert len(host_batches) == len(dev_batches) > 0
    for (hx, hy), (dx, dy) in zip(host_batches, dev_batches):
        assert isinstance(dx, images.PackedRegions) and len(dx) == hx.shape[0]
        assert torch.equal(hy, dy)
        twin = images.resized_crop_reference(dx.data, dx.desc, size)
        levels = ((twin - hx.double()) * 255).abs().max().item()
        assert levels <= PIL_LEVELS, levels


@pytest.mark.parametrize("num_workers", [0, 2])
def test_image_folder_same_crops_and_flips(tmp_path, num_workers):
    root = _folder(str(tmp_path / "train"))
    for train in (True, False):
        got = {}
        for augment in ("host", "device"):
            torch.manual_seed(7)
            loader, _ = images.image_folder_loader(root, 4, train, 224, num_workers, device_normalize=True,
                                                   augment=augment)
            got[augment] = list(loader)
        _compare(got["host"], got["device"], 224)


@pytest.mark.parametrize("num_workers", [0, 2])
def test_record_loader_same_crops_and_flips(tmp_path, num_workers):
    root = _folder(str(tmp_path / "train"))
    files, labels, _ = records.find_image_files(root)
    out = str(tmp_path / "rec")
    assert records.write_shards(files, labels, out, "train", 2) == len(files)
    for train in (True, False):
        got = {}
        for augment in ("host", "device"):
            torch.manual_seed(11)
            loader = records.RecordLoader(out, "train", 4, train, 224, num_workers, normalize_on_host=False, seed=3,
                                          augment=augment)
            loader.set_epoch(1)
            got[augment] = list(loader)
        _compare(got["host"], got["device"], 224)


def test_collate_packs_aligned_regions():
    rng = np.random.default_rng(0)
    regions = [rng.integers(0, 256, (h, w, 3), dtype=np.uint8) for h, w in ((5, 7), (1, 1), (16, 3), (9, 11))]
    descs = [(r.shape[0], r.shape[1], r.shape[0] / 224, r.shape[1] / 224, 0, 0, k % 2) for k, r in enumerate(regions)]
    packed, labels = images.collate_regions([((r, d), k) for k, (r, d) in enumerate(zip(regions, descs))])
    assert labels.tolist() == [0, 1, 2, 3]
    assert packed.data.dtype == torch.uint8 and packed.data.dim() == 1
    assert packed.desc.dtype == torch.float64 and packed.desc.shape == (4, 8)
    offsets = [int(o) for o in packed.desc[:, 0]]
    assert offsets == [0, 112, 128, 272]                  # 105 -> 112, 3 -> 16, 144 -> 144 bytes: 16-byte aligned
    assert packed.data.numel() >= offsets[-1] + regions[-1].size
    for r, d, off, row in zip(regions, descs, offsets, packed.desc.tolist()):
        assert off % 16 == 0 and row[1:] == list(map(float, d))
        assert np.array_equal(packed.data[off:off + r.size].numpy(), r.reshape(-1))
    native.check_resized_crop_desc(packed.desc, packed.data.numel(), 224)
    moved = packed.to("cpu")
    assert moved.data is packed.data and moved.desc is packed.desc


def _good():
    return torch.tensor([[0, 10, 20, 10 / 224, 20 / 224, 0, 0, 0], [608, 30, 40, 20 / 224, 30 / 224, 5, 7, 1]],
                        dtype=torch.float64)


@pytest.mark.parametrize("case", [
    "offset_past_end", "negative_offset", "fractional_offset", "zero_height", "zero_width", "zero_scale",
    "negative_scale", "nan_scale", "inf_scale", "flip_2", "negative_crop_offset", "crop_offset_past_region",
    "float32_desc", "wrong_width"])
def test_malformed_descriptors_are_refused(case):
    n = 608 + 30 * 40 * 3
    native.check_resized_crop_desc(_good(), n, 224)
    d = _good()
    edits = {"offset_past_end": (1, 0, 609.0), "negative_offset": (0, 0, -16.0), "fractional_offset": (1, 0, 608.5),
             "zero_height": (0, 1, 0.0), "zero_width": (1, 2, 0.0), "zero_scale": (0, 3, 0.0),
             "negative_scale": (1, 4, -1.0), "nan_scale": (0, 3, float("nan")), "inf_scale": (1, 4, float("inf")),
             "flip_2": (1, 7, 2.0), "negative_crop_offset": (1, 5, -1.0), "crop_offset_past_region": (1, 6, 1000.0)}
    if case in edits:
        i, j, v = edits[case]
        d[i, j] = v
    elif case == "float32_desc":
        d = d.float()
    else:
        d = d[:, :7]
    with pytest.raises(ValueError):
        native.check_resized_crop_desc(d, n, 224)


def test_resized_crop_refuses_host_data():
    d = _good()
    m = torch.zeros(3)
    with pytest.raises(ValueError):
        native.resized_crop(torch.zeros(608 + 3600, dtype=torch.uint8), d, 224, m, m)


def test_imagenet_trainer_refusals(tmp_path):
    from distributeddeeplearning_b200.workloads import imagenet

    with pytest.raises(ValueError, match="real data"):
        imagenet.main(use_gpu=True, augment="device", epochs=0)
    with pytest.raises(ValueError, match="host or device"):
        imagenet.main(augment="gpu", epochs=0)
    if not torch.cuda.is_available():
        with pytest.raises(ValueError, match="use_gpu"):
            imagenet.main(training_data_path=str(tmp_path), use_gpu=True, augment="device", epochs=0)
        with pytest.raises(ValueError, match="use_gpu"):
            imagenet.main(training_data_path=str(tmp_path), data_type="records", augment="device", epochs=0)


def test_hvd_trainer_refusals(tmp_path):
    from distributeddeeplearning_b200.workloads import hvd_imagenet

    with pytest.raises(ValueError, match="real data"):
        hvd_imagenet.main(["--augment", "device"])
    with pytest.raises(ValueError, match="CUDA"):
        hvd_imagenet.main(["--augment", "device", "--no-cuda", "--train-dir", str(tmp_path)])
    with pytest.raises(SystemExit):
        hvd_imagenet.main(["--augment", "gpu"])


def test_loaders_refuse_unknown_augment(tmp_path):
    with pytest.raises(ValueError):
        images.image_folder_loader(str(tmp_path), 4, True, augment="gpu")


def test_tasks_forward_augment(monkeypatch):
    from distributeddeeplearning_b200.cli import tasks

    calls = []
    monkeypatch.setattr(tasks, "_submit", lambda module, argv, *a, **k: calls.append(list(argv)))
    monkeypatch.setattr(tasks, "_env", lambda: {"DATA": "/data"})
    monkeypatch.setattr(tasks, "_datastore_path", lambda: "/store")
    for fn in (tasks.imagenet_images_local, tasks.imagenet_records_local):
        fn.body(None, augment="device")
        fn.body(None)
    tasks.imagenet_images_remote.body(None, node_count=1, augment="device")
    tasks.imagenet_records_remote.body(None, node_count=1, augment="device")
    tasks.hvd_images_remote.body(None, node_count=1, augment="device")
    for argv, device in zip(calls, (True, False, True, False, True, True, True)):
        assert (argv[argv.index("--augment") + 1] == "device") if device else "--augment" not in argv, argv


def _ptxas(src):
    """{demangled kernel name: (registers, spill store bytes, spill load bytes)} of one .cu file built for sm_90a."""
    nvcc = os.path.join(_ext.CUDA_HOME, "bin", "nvcc")
    csrc = os.path.join(os.path.dirname(_ext.__file__), "csrc")
    r = subprocess.run([nvcc, "-c", os.path.join(csrc, "ops", src), "-o", os.devnull, "-O3", "-std=c++17", *_ext.NVCC_ARCH,
                        "--expt-relaxed-constexpr", "-I", csrc, "-Xptxas", "-v"], capture_output=True, text=True)
    assert r.returncode == 0, r.stderr[-3000:]
    out, cur = {}, None
    for line in r.stderr.splitlines():
        m = re.search(r"Function properties for (\S+)", line)
        if m:
            cur = subprocess.run(["c++filt", m.group(1)], capture_output=True, text=True).stdout.strip()
            cur = re.sub(r"^(void )?ddl::|\(.*\)$", "", cur.replace("(anonymous namespace)::", ""))
            continue
        m = re.search(r"(\d+) bytes spill stores, (\d+) bytes spill loads", line)
        if m and cur:
            out[cur] = [0, int(m.group(1)), int(m.group(2))]
        m = re.search(r"Used (\d+) registers", line)
        if m and cur:
            out[cur][0] = int(m.group(1))
    return out


_NVCC = shutil.which("c++filt") and os.path.isfile(os.path.join(_ext.CUDA_HOME, "bin", "nvcc"))


@pytest.mark.skipif(not _NVCC, reason="needs nvcc and c++filt")
def test_augment_kernel_compiles_without_spills():
    k = _ptxas("augment.cu")
    assert sorted(k) == ["resized_crop_kernel"], sorted(k)
    regs, st, ld = k["resized_crop_kernel"]
    assert st == 0 and ld == 0, (regs, st, ld)
    assert regs <= 128, regs                     # __launch_bounds__(128): no register cap below 255 is forced


def test_resized_crop_is_counted():
    assert _ext.KERNEL_LAUNCHES["resized_crop"] == 1
    src = open(os.path.join(os.path.dirname(_ext.__file__), "csrc", "ops", "augment.cu")).read()
    assert "<<<" not in src and not re.search(r"atomic[A-Z]\w*\(", src) and src.count("launch_pdl(") == 1
