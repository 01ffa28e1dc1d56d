"""In-tree build + loader of the native module ``distributeddeeplearning_b200._C``.

* ``build()``  compiles every ``csrc/**/*.cu`` with
  ``nvcc -gencode arch=compute_90a,code=sm_90a -lineinfo`` (cross-compiles without a GPU),
  every ``csrc/**/*.cpp`` with g++, and links ``_C.so`` next to this file (so the artefact
  travels with the source tree and shows up as an in-tree native module).
* ``load()``   imports ``_C``; (re)builds first when the sources are newer than the artefact.
  There is no eager-PyTorch fallback for GPU execution: if a CUDA device is present and the module
  cannot be loaded, ``load()`` raises.
"""
from __future__ import annotations

import hashlib
import importlib
import os
import subprocess
import sys
import sysconfig
import threading
from concurrent.futures import ThreadPoolExecutor
from typing import List, Optional

_HERE = os.path.dirname(os.path.abspath(__file__))
_CSRC = os.path.join(_HERE, "csrc")
_BUILD = os.path.join(_HERE, "csrc", "build")
_SO = os.path.join(_HERE, "_C.so")
_STAMP = os.path.join(_BUILD, "sources.sha")
_LOCK = threading.Lock()
_MODULE = None

NVCC_ARCH = ["-gencode", "arch=compute_90a,code=sm_90a"]
CUDA_HOME = os.environ.get("CUDA_HOME", "/usr/local/cuda")


def _sources() -> List[str]:
    out = []
    for root, _dirs, files in os.walk(_CSRC):
        if os.path.abspath(root).startswith(os.path.abspath(_BUILD)):
            continue
        for f in sorted(files):
            if f.endswith((".cu", ".cpp")):
                out.append(os.path.join(root, f))
    return sorted(out)


def _all_inputs() -> List[str]:
    out = []
    for root, _dirs, files in os.walk(_CSRC):
        if os.path.abspath(root).startswith(os.path.abspath(_BUILD)):
            continue
        for f in sorted(files):
            if f.endswith((".cu", ".cpp", ".cuh", ".h")):
                out.append(os.path.join(root, f))
    return sorted(out)


def _digest() -> str:
    h = hashlib.sha256()
    for p in _all_inputs():
        h.update(os.path.relpath(p, _CSRC).encode())
        with open(p, "rb") as f:
            h.update(f.read())
    return h.hexdigest()


def is_stale() -> bool:
    if not os.path.isfile(_SO) or not os.path.isfile(_STAMP):
        return True
    try:
        with open(_STAMP) as f:
            return f.read().strip() != _digest()
    except OSError:
        return True


class _build_lock:
    """Cross-process lock around the build (all ranks of a job import the package at once; if the module were stale they
    would otherwise compile into the same build directory concurrently)."""

    def __enter__(self):
        import fcntl

        os.makedirs(_BUILD, exist_ok=True)
        self.f = open(os.path.join(_BUILD, ".lock"), "w")
        fcntl.flock(self.f, fcntl.LOCK_EX)
        return self

    def __exit__(self, *exc):
        import fcntl

        fcntl.flock(self.f, fcntl.LOCK_UN)
        self.f.close()
        return False


def _pybind_include() -> str:
    import pybind11

    return pybind11.get_include()


def _run(cmd: List[str], verbose: bool) -> None:
    if verbose:
        print(" ".join(cmd), flush=True)
    r = subprocess.run(cmd, capture_output=True, text=True)
    if r.returncode != 0:
        raise RuntimeError("build command failed:\n" + " ".join(cmd) + "\n" + r.stdout + r.stderr)
    if verbose and (r.stdout or r.stderr):
        print(r.stdout + r.stderr, flush=True)


def build(verbose: bool = False, force: bool = False, ptxas_info: bool = False) -> str:
    """Compile and link ``_C.so``; returns its path."""
    with _LOCK, _build_lock():
        # (the file lock serialises the ranks of one job: whoever gets it first builds, the others find a fresh module)
        if not force and not is_stale():
            return _SO
        nvcc = os.path.join(CUDA_HOME, "bin", "nvcc")
        if not os.path.isfile(nvcc):
            raise RuntimeError(f"nvcc not found at {nvcc}; cannot build the native module")
        os.makedirs(_BUILD, exist_ok=True)
        py_inc = sysconfig.get_paths()["include"]
        common_inc = ["-I", _CSRC, "-I", os.path.join(CUDA_HOME, "include"), "-I", py_inc, "-I", _pybind_include()]
        objs, jobs = [], []
        for src in _sources():
            rel = os.path.relpath(src, _CSRC).replace(os.sep, "_")
            obj = os.path.join(_BUILD, rel + ".o")
            objs.append(obj)
            if src.endswith(".cu"):
                cmd = [nvcc, "-c", src, "-o", obj, "-O3", "-std=c++17", "-lineinfo", *NVCC_ARCH,
                       "-Xcompiler", "-fPIC", "--expt-relaxed-constexpr", "-Xcompiler", "-fvisibility=hidden",
                       *common_inc]
                if ptxas_info:
                    cmd += ["-Xptxas", "-v"]
            else:
                cmd = ["g++", "-c", src, "-o", obj, "-O2", "-std=c++17", "-fPIC", "-fvisibility=hidden",
                       "-pthread", *common_inc]
            jobs.append(cmd)
        with ThreadPoolExecutor(max_workers=min(8, len(jobs))) as ex:
            list(ex.map(lambda c: _run(c, verbose), jobs))
        link = ["g++", "-shared", "-o", _SO + ".tmp", *objs, "-L", os.path.join(CUDA_HOME, "lib64"), "-lcudart",
                "-ldl", "-lpthread", "-Wl,-rpath," + os.path.join(CUDA_HOME, "lib64")]
        _run(link, verbose)
        os.replace(_SO + ".tmp", _SO)
        with open(_STAMP, "w") as f:
            f.write(_digest())
        return _SO


# kernels launched per call of each binding (everything not listed launches none)
KERNEL_LAUNCHES = {
    "fused_sgd_local": 1, "fused_allreduce_sgd": 1, "allreduce": 1, "broadcast": 1, "barrier": 1,
    "allgather_slices": 1, "conv_gemm": 1, "conv_wgrad": 1, "bn_act_fwd": 1, "bn_act_bwd": 2, "channel_stats": 1,
    "maxpool_fwd": 1, "maxpool_bwd": 1, "avgpool_fwd": 1, "avgpool_bwd": 1, "global_avgpool_fwd": 1,
    "global_avgpool_bwd": 1, "softmax_xent": 1, "philox_normal_nhwc": 1, "philox_labels": 1, "nchw_to_nhwc_norm": 1,
    "nhwc_u8_to_nhwc4": 1, "cast_f32_bf16": 1, "pack_stem_weight": 1, "unpack_stem_grad": 1, "bias_relu_bwd": 1,
    "dropout": 1, "add_bf16": 1, "fp8_quantize": 1, "fp8_quantize_mx": 1, "fp8_transpose_taps": 1, "fp8_amax": 1, "fp8_update_scales": 1, "pad_nhwc4": 1, "expand_grouped_weight": 1, "concat_channels": 1, "bn_relu_maxpool_fwd": 1, "bn_pool_bwd": 2,
    "dwconv_fwd": 1, "dwconv_dgrad": 1, "dwconv_wgrad": 1, "se_scale": 1, "se_reduce": 1, "se_apply": 1,
    "hardswish_fwd": 1, "hardswish_bwd": 1, "se_sig_scale": 1, "se_sig_reduce": 1, "se_sig_apply": 1, "pad_cols": 1,
    "fold_cols": 1, "silu_rows_fwd": 1, "silu_rows_bwd": 1, "stochastic_depth_keep": 1,
    "dwconv7_fwd": 1, "dwconv7_dgrad": 1, "dwconv7_wgrad": 1, "layer_norm_fwd": 1, "layer_norm_bwd": 1, "gelu_fwd": 1,
    "gelu_bwd": 1, "layer_scale_fwd": 1, "layer_scale_bwd": 1,
    "attention_fwd": 1, "attention_bwd": 2, "add_layer_norm_fwd": 1, "layer_norm_bwd_add": 1, "patchify": 1,
    "tokens_fwd": 1, "tokens_bwd": 2,
    "window_attention_fwd": 1, "window_attention_bwd": 3, "patch_merge_fwd": 1, "patch_merge_bwd": 2,
    "window_attention_v2_fwd": 1, "window_attention_v2_bwd": 3, "cpb_fwd": 1, "cpb_bwd": 2, "merge_gather": 1,
    "grid_attention_fwd": 1, "grid_attention_bwd": 3, "tanh_rows_fwd": 1, "tanh_rows_bwd": 1,
    "shuffle_fwd": 1, "shuffle_bwd": 2,
    "bn_seg_fwd": 1, "bn_seg_bwd": 2, "adaptive_avgpool_fwd": 1, "adaptive_avgpool_bwd": 1, "transpose_rows": 1,
    "resized_crop": 1,
}
LAUNCH_COUNT = [0]          # kernels of THIS repo launched so far (bench.py reports the per-region delta)


class _Counting:
    """Thin proxy over ``_C`` that counts kernel launches of this repo's own kernels."""

    def __init__(self, mod):
        self._mod = mod
        for name in dir(mod):
            if name.startswith("__"):
                continue
            obj = getattr(mod, name)
            n = KERNEL_LAUNCHES.get(name)
            if n and callable(obj):
                setattr(self, name, self._wrap(obj, n))
            else:
                setattr(self, name, obj)

    @staticmethod
    def _wrap(fn, n):
        def call(*a, **kw):
            LAUNCH_COUNT[0] += n
            return fn(*a, **kw)
        call.__name__ = getattr(fn, "__name__", "kernel")
        return call


def launch_count() -> int:
    return LAUNCH_COUNT[0]


def add_launches(n: int) -> None:
    """Account for kernels launched by replaying a captured CUDA graph (the bindings are not called on replay)."""
    LAUNCH_COUNT[0] += int(n)


def load(auto_build: bool = True):
    """Import the native module (building it first if needed)."""
    global _MODULE
    if _MODULE is not None:
        return _MODULE
    if auto_build and is_stale():
        nvcc = os.path.join(CUDA_HOME, "bin", "nvcc")
        if os.path.isfile(nvcc):
            build()
        elif not os.path.isfile(_SO):
            raise RuntimeError("native module _C.so is missing and nvcc is unavailable to build it")
    import torch  # noqa: F401  (loads libcudart.so.12 that _C.so links against)

    _MODULE = _Counting(importlib.import_module("distributeddeeplearning_b200._C"))
    return _MODULE


def available() -> bool:
    try:
        load()
        return True
    except Exception:
        return False


def sass(pattern: Optional[str] = None) -> str:
    """cuobjdump -sass of the built module (profiling evidence helper)."""
    cuobjdump = os.path.join(CUDA_HOME, "bin", "cuobjdump")
    r = subprocess.run([cuobjdump, "-sass", _SO], capture_output=True, text=True)
    txt = r.stdout
    if pattern:
        import re

        txt = "\n".join(line for line in txt.splitlines() if re.search(pattern, line))
    return txt


if __name__ == "__main__":
    path = build(verbose=True, force="--force" in sys.argv, ptxas_info="--ptxas" in sys.argv)
    print("built", path)
