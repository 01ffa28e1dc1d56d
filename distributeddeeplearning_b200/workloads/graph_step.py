"""Whole-step CUDA-graph capture / replay shared by the workloads.

A training step of this framework is ~340 kernel launches on three streams (main, weight-gradient side stream,
bucket/comm stream) plus the Python autograd walk; at the reference's default batch of 64 images per GPU the host
cannot issue them as fast as one H100 retires them.  ``GraphedStep`` captures ``fn(*static_inputs)`` once (after
warm-up) and replays it: per step the host copies the new inputs into the static buffers, refreshes the pinned
hyper-parameter blob (so LR schedules keep working — the upload is a memcpy node of the graph) and issues a single
``cudaGraphLaunch``.

Capture rules the framework follows (see DESIGN.md 4.1): accumulators come from an arena whose memset is the first
graph node (``native.begin_capture_scratch``); streams only join what is pending (``functional.wgrad_join``); dropout
masks stay fresh because their Philox key mixes in a device-resident step counter that the captured step increments
(``ops.advance_dropout_step``) — launch arguments such as the host-side offset are frozen by a graph.
"""
from __future__ import annotations

from typing import Callable, Optional, Sequence, Tuple

import torch

from .. import ops


def model_has_dropout(model: torch.nn.Module) -> bool:
    for m in [model] + list(model.modules()):
        p = getattr(m, "p", None)
        if isinstance(p, (int, float)) and float(p) > 0.0:
            return True
    return False


class GraphedStep:
    """``fn(*inputs) -> tensor | tuple of tensors`` replayed from a CUDA graph for inputs of the captured shapes."""

    def __init__(self, fn: Callable, optimizer, log: Optional[Callable[[str], None]] = None,
                 capture_error_mode: str = "global"):
        """``capture_error_mode``: torch's mode for the capture.  ``thread_local`` for callers whose DataLoader runs a
        pin-memory thread: that thread allocates pinned buffers (``cudaHostAlloc``) while the step is captured, which
        the default ``global`` mode makes fail as an unsafe call from another thread (DESIGN.md 4.1)."""
        def stepped(*inputs):
            out = fn(*inputs)
            ops.advance_dropout_step()          # part of the captured step: replays draw fresh dropout masks
            return out

        self.fn, self.optimizer, self.log = stepped, optimizer, log or (lambda s: None)
        self.graph = None
        self.static_in: Tuple[torch.Tensor, ...] = ()
        self.static_out = None
        self.launches = 0
        self.failed = False
        self.capture_error_mode = capture_error_mode

    @staticmethod
    def applicable(model: torch.nn.Module, optimizer, example: torch.Tensor) -> bool:
        from ..parallel.engine import FusedSGD

        return bool(example.is_cuda and isinstance(optimizer, FusedSGD) and ops.use_native(example))

    def capture(self, inputs: Sequence[torch.Tensor], warmup: int = 3) -> bool:
        """Warm up eagerly on ``inputs`` (kernel configuration, momentum init, allocator), then capture one step."""
        from .. import _ext
        from ..ops import native

        for _ in range(max(1, warmup)):
            self.fn(*inputs)
        torch.cuda.synchronize()
        self.static_in = tuple(t.clone() for t in inputs)
        graph = torch.cuda.CUDAGraph()
        before = _ext.launch_count()
        try:
            with torch.cuda.graph(graph, capture_error_mode=self.capture_error_mode):
                native.begin_capture_scratch(self.static_in[0].device)
                self.static_out = self.fn(*self.static_in)
        except Exception as e:  # stay eager, say why
            native.end_capture_scratch()
            self.failed = True
            self.log("CUDA graph capture failed (%s); staying eager" % (str(e).splitlines()[0],))
            torch.cuda.synchronize()
            return False
        native.end_capture_scratch()
        self.launches = _ext.launch_count() - before
        self.graph = graph
        return True

    def matches(self, inputs: Sequence[torch.Tensor]) -> bool:
        return self.graph is not None and len(inputs) == len(self.static_in) and all(
            a.shape == b.shape and a.dtype == b.dtype for a, b in zip(inputs, self.static_in))

    def __call__(self, *inputs: torch.Tensor):
        """Replay for matching shapes (e.g. every full batch), run ``fn`` eagerly otherwise (a short last batch)."""
        if not self.matches(inputs):
            return self.fn(*inputs)
        from .. import _ext

        for src, dst in zip(inputs, self.static_in):
            if src is not dst:
                dst.copy_(src, non_blocking=True)
        if hasattr(self.optimizer, "refresh_hyper_host"):
            self.optimizer.refresh_hyper_host()
        self.graph.replay()
        if hasattr(self.optimizer, "mark_hyper_consumed"):
            self.optimizer.mark_hyper_consumed()       # the replay's memcpy node read the pinned hyper blob
        _ext.add_launches(self.launches)
        return self.static_out
