"""FP8 training mode: e4m3 activations / weights and e5m2 gradients as tensor-core operands of the forward and
data-gradient convolutions (``wgmma ... .e4m3.e4m3`` / ``.e5m2.e4m3``), everything else unchanged (bf16 activations in
memory, fp32 accumulation, bf16 weight-gradient GEMMs, fp32 BN / softmax / master weights / optimizer).  fp8 wgmma reads
K-major operands only, so the data gradient takes its weights from a per-step transposed e4m3 copy
``[Cin][R*S*Cout]`` (``quantize_weight_t``) instead of reading the forward's copy MN-major.

Reference parity: the only reduced-precision switch the reference has is ``--use_fp16`` of its TensorFlow benchmark
tasks (``TensorFlow_benchmark/tensorflow_benchmark.py:51,77``); on Hopper the equivalent "use the fast tensor-core
format" switch is FP8 (BASELINE config #3).  Enabled with ``--precision fp8`` on the trainers / ``DDL_PRECISION=fp8``.

Recipe = delayed per-tensor scaling (csrc/ops/fp8.cu): each quantised tensor role owns a slot {amax, scale,
inv_scale} in ONE device table; quantisation multiplies by the slot's power-of-two scale and records the amax that
becomes next step's scale (``end_of_step`` = one tiny kernel for the whole model, part of the captured CUDA graph).
Layers whose reduction dimension is not a multiple of 128 channels (the stem, layer1's 64-channel convs) and the
classifier stay in bf16 — the usual "first and last layer in higher precision" rule falls out of the geometry.
"""
from __future__ import annotations

import os
from typing import Dict, Optional, Tuple

import torch

from .. import _ext

_STATE = {"enabled": os.environ.get("DDL_PRECISION", "bf16").lower() == "fp8", "table": None, "n": 0, "slots": {},
          "calibrated": set(), "step": 0, "wcache": {}, "stats": {"fwd": 0, "dgrad": 0}}
_MAX_SLOTS = 4096


def enable(on: bool = True) -> None:
    _STATE["enabled"] = bool(on)


def enabled() -> bool:
    return bool(_STATE["enabled"])


def launches() -> Dict[str, int]:
    """How many forward / dgrad launches took the fp8 path so far (tests assert the mode is really exercised)."""
    return dict(_STATE["stats"])


def _table(device) -> torch.Tensor:
    t = _STATE["table"]
    if t is None:
        C = _ext.load()
        assert int(C.FP8_SLOT_BYTES) == 16
        t = torch.zeros((_MAX_SLOTS, 4), dtype=torch.float32, device=device)
        t[:, 1] = 1.0          # scale
        t[:, 2] = 1.0          # inv_scale
        _STATE["table"] = t
    return t


def _slot(key, device, e5m2: bool) -> int:
    """Index of the slot of tensor role ``key`` (allocated on first use)."""
    s = _STATE["slots"].get(key)
    if s is None:
        if _STATE["n"] >= _MAX_SLOTS:
            raise RuntimeError("fp8: slot table full")
        s = _STATE["n"]
        _STATE["n"] += 1
        _STATE["slots"][key] = s
        if e5m2:
            _table(device)[s, 3] = 1.0        # Fp8Slot::e5m2 != 0 (the kernel only tests the field for non-zero)
    return s


def slot_ptr(idx: int, device) -> int:
    return _table(device).data_ptr() + 16 * idx


def inv_scale_ptr(idx: int, device) -> int:
    return slot_ptr(idx, device) + 8


def quantize(x: torch.Tensor, key, e5m2: bool = False) -> Tuple[torch.Tensor, int]:
    """bf16 tensor (any layout, quantised in memory order) -> (uint8 tensor of fp8 codes, slot index)."""
    from . import native

    C = _ext.load()
    dev = x.device
    idx = _slot(key, dev, e5m2)
    st = torch.cuda.current_stream(dev).cuda_stream
    sms = native.sm_count(dev.index or 0)
    n = x.numel()
    if idx not in _STATE["calibrated"]:
        if torch.cuda.is_current_stream_capturing():
            raise RuntimeError("fp8: a tensor role was first seen during CUDA-graph capture (warm up eagerly first)")
        # first use: measure amax now and derive the scale from it, so step 0 is not quantised blindly
        C.fp8_amax(x.data_ptr(), n, slot_ptr(idx, dev), sms, st)
        C.fp8_update_scales(slot_ptr(idx, dev), 1, st)
        _STATE["calibrated"].add(idx)
    out = torch.empty_like(x, dtype=torch.uint8)       # same strides: NHWC stays NHWC
    C.fp8_quantize(x.data_ptr(), out.data_ptr(), n, slot_ptr(idx, dev), e5m2, sms, st)
    return out, idx


# ---- producer-side quantisation ("twins") -------------------------------------------------------------------------
# The BN-apply kernels can emit the fp8 copy of their output in the same streaming pass (bn_act.cu, FP8 variants): the
# producer registers it here, the consuming convolution looks it up by tensor identity and skips its own quantise pass.
# Entries hold a weak reference to the bf16 tensor (a recycled address can never alias) and die at the end of the step.
import weakref

_TWINS = {}
_PRODUCED = {}        # id(bf16 tensor) -> (weakref, producer key): who wrote this tensor (this step)
_WANTED = set()       # producer keys whose output an fp8 convolution actually consumes: only those emit a twin


def note_producer(t: torch.Tensor, key) -> bool:
    """Called by a kernel wrapper that COULD emit a twin of ``t``; returns whether a consumer asked for one."""
    _PRODUCED[id(t)] = (weakref.ref(t), key)
    return key in _WANTED


def request_twin(t: torch.Tensor) -> None:
    """Called by an fp8 convolution that had to quantise ``t`` itself: from the next step on its producer does it."""
    e = _PRODUCED.get(id(t))
    if e is not None and e[0]() is t:
        _WANTED.add(e[1])


def producer_slot(key, device, like: torch.Tensor, e5m2: bool = False):
    """(slot index, fused) for a tensor role quantised by its producing kernel.  ``fused`` is False until the slot is
    calibrated: the first time the producer runs plain and ``attach_by_quantize`` does the two-pass calibration."""
    idx = _slot(key, device, e5m2)
    return idx, idx in _STATE["calibrated"]


def attach_twin(t: torch.Tensor, q: torch.Tensor, idx: int) -> None:
    _TWINS[id(t)] = (weakref.ref(t), q, idx)


def attach_by_quantize(t: torch.Tensor, key, e5m2: bool = False) -> None:
    q, idx = quantize(t, key, e5m2)
    attach_twin(t, q, idx)


def twin_of(t: torch.Tensor):
    e = _TWINS.get(id(t))
    if e is None or e[0]() is not t:
        return None
    return e[1], e[2]


def quantize_weight(w_bf16: torch.Tensor) -> Tuple[torch.Tensor, int]:
    """e4m3 copy of a bf16 weight matrix, quantised once per step and shared by forward and dgrad."""
    key = ("w", w_bf16.data_ptr(), tuple(w_bf16.shape))
    hit = _STATE["wcache"].get(key)
    if hit is not None and hit[0] == _STATE["step"]:
        return hit[1], hit[2]
    q, idx = quantize(w_bf16, key)
    _STATE["wcache"][key] = (_STATE["step"], q, idx)
    return q, idx


def quantize_weight_t(w_bf16: torch.Tensor, taps: int, cin: int) -> Tuple[torch.Tensor, int]:
    """The data gradient's K-major e4m3 weights: this step's copy of ``w_bf16`` [Cout][taps*Cin] transposed to
    [Cin][taps*Cout] (same codes, same scale slot), made once per step."""
    q, idx = quantize_weight(w_bf16)
    key = ("wt", w_bf16.data_ptr(), tuple(w_bf16.shape))
    hit = _STATE["wcache"].get(key)
    if hit is not None and hit[0] == _STATE["step"]:
        return hit[1], hit[2]
    cout = w_bf16.shape[0]
    qt = torch.empty((cin, taps * cout), dtype=torch.uint8, device=w_bf16.device)
    _ext.load().fp8_transpose_taps(q.data_ptr(), qt.data_ptr(), cout, taps, cin,
                                   torch.cuda.current_stream(w_bf16.device).cuda_stream)
    _STATE["wcache"][key] = (_STATE["step"], qt, idx)
    return qt, idx


def end_of_step(device=None) -> None:
    """amax -> next step's scale for every slot (one launch); called by the optimizers' ``step()``."""
    if not _STATE["enabled"] or _STATE["table"] is None or _STATE["n"] == 0:
        return
    t = _STATE["table"]
    C = _ext.load()
    C.fp8_update_scales(t.data_ptr(), int(_STATE["n"]), torch.cuda.current_stream(t.device).cuda_stream)
    _TWINS.clear()
    _PRODUCED.clear()
    _STATE["step"] += 1          # next step quantises its weights again (a captured step never reuses an eager copy)


# fp8 pays where the main loop dominates (long reductions); short ones are epilogue-bound.  The 512-element threshold
# was not re-measured on H100.
MIN_K = int(os.environ.get("DDL_FP8_MIN_K", "512"))


def fwd_eligible(cin: int, cout: int, taps: int = 1) -> bool:
    return _STATE["enabled"] and cin % 128 == 0 and cout % 64 == 0 and cin * taps >= MIN_K


def dgrad_eligible(cin: int, cout: int, taps: int = 1) -> bool:
    # reduction dim = Cout (k-blocks of 128), transposed weight rows = input channels (N tiles of 128)
    return _STATE["enabled"] and cout % 128 == 0 and cin % 128 == 0 and cout * taps >= MIN_K


def count(kind: str) -> None:
    _STATE["stats"][kind] += 1


def reset() -> None:
    """Forget all slots (tests)."""
    _STATE.update(table=None, n=0, slots={}, calibrated=set(), step=0, wcache={}, stats={"fwd": 0, "dgrad": 0})
    _TWINS.clear()
    _PRODUCED.clear()
    _WANTED.clear()
