"""Checked Python wrappers over the sm_90a kernels in ``_C`` (GPU only).

Activations are ``torch.bfloat16`` tensors with logical shape ``[N, C, H, W]`` and
``channels_last`` memory (physically NHWC).  Convolution weights are logical
``[Cout, Cin, R, S]`` ``channels_last`` (physically KRSC), which is exactly the row-major
``[Cout][R*S*Cin]`` GEMM operand the wgmma kernels consume — the bf16 compute copy is a flat
cast of the fp32 master, and wgrad writes the fp32 gradient in the same layout.
"""
from __future__ import annotations

import functools
import os
from typing import Optional, Tuple

import torch

from .. import _ext

CL = torch.channels_last


@functools.lru_cache(maxsize=None)
def _C():
    C = _ext.load()
    if os.environ.get("DDL_WGRAD_SWAP", "1") == "0":       # tuning hook (A/B runs): no operand-role swap in wgrad
        C.set_wgrad_swap(0)
    if os.environ.get("DDL_CONV_PERSISTENT", "") in ("0", "2"):    # tuning hook: 0 = never, 2 = always persistent
        C.set_conv_persistent(int(os.environ["DDL_CONV_PERSISTENT"]))
    if os.environ.get("DDL_CONV_CLUSTER", "0") in ("1", "2"):     # tuning hook: the persistent kernel as CTA pairs that
        C.set_conv_cluster(int(os.environ["DDL_CONV_CLUSTER"]))       #   share the weight tile by TMA multicast
    if os.environ.get("DDL_BN_REVERSE", "") in ("0", "1"):             # BN row traversal order (A/B runs)
        C.set_bn_reverse(int(os.environ["DDL_BN_REVERSE"]))
    if os.environ.get("DDL_CONV_WAIT_HINT", ""):                       # ns; suspend-time hint of the mbarrier waits (A/B runs)
        C.set_conv_wait_hint(int(os.environ["DDL_CONV_WAIT_HINT"]))
    if os.environ.get("DDL_PDL", "") in ("0", "1", "2", "3"):         # programmatic dependent launch (A/B runs, launch.h)
        C.set_pdl(int(os.environ["DDL_PDL"]))
    if os.environ.get("DDL_CONV_DEEP", "") in ("0", "2", "3", "4"):   # 2 = persistent CTA pairs wherever they apply,
        C.set_conv_deep(int(os.environ["DDL_CONV_DEEP"]))            #   3 / 4 = persistent single CTAs
    return C


# ------------------------------------------------------------------------------------------------
# per-shape kernel autotuning — the analogue of the reference's ``torch.backends.cudnn.benchmark = True``
# (``PyTorch_benchmark/src/pytorch_synthetic_benchmark.py:57``, ``PyTorch_imagenet/src/imagenet_pytorch_horovod.py:378``)
# ------------------------------------------------------------------------------------------------
# The launcher (csrc/ops/conv_gemm.cu) has several kernels for the same maths (one tile per CTA; persistent with one
# CTA per SM walking tiles; the persistent kernel as CTA pairs sharing the weight tile by TMA multicast).  Which one wins
# depends on K, the number of tiles and how memory-bound the epilogue is, so the first (eager) call of every distinct
# layer shape times the applicable variants on the real operands and remembers the winner; CUDA-graph capture and all
# later calls use the table.  ``DDL_CONV_AUTOTUNE=0`` keeps the launcher's built-in policy.
VAR_ONE_TILE, VAR_PERSISTENT = 1, 2
VAR_PAIR = 1 << 8
_TUNE = {"enabled": os.environ.get("DDL_CONV_AUTOTUNE", "1") == "1", "table": {}, "timings": {}}


def conv_variants(n_total: int, m_rows: int, kb: int, b_mn_major: bool, fp8: bool = False, grouped: bool = False):
    """Variant words worth timing for an ``m_rows`` x ``n_total`` x ``kb*64`` problem (see launch_fwd_mode).  fp8
    operands run on the one-tile kernel only; grouped tiles are 64 wide."""
    out = [VAR_ONE_TILE]
    if fp8 or m_rows < 128 * 132:     # less than one wave of 128-row tiles: the persistent kernels cannot pay
        return out
    out.append(VAR_PERSISTENT)
    if not (b_mn_major and (n_total % 128 != 0 or grouped)):   # MN-major weight tiles split into two 64-column boxes
        out.append(VAR_PERSISTENT | VAR_PAIR)
    return out


def force_variant(v: Optional[int]) -> None:
    """Tools / tests: make every tunable conv launch use variant ``v`` (None = back to autotuning)."""
    _TUNE["force"] = v


def variant_name(v: int) -> str:
    return {0: "policy", 1: "one-tile", 2: "persistent"}[v & 0xf] + ("-pair" if v & VAR_PAIR else "")


def autotune_table():
    """{shape key: (chosen variant name, {variant name: microseconds})} — what the tuner decided so far."""
    return {k: (variant_name(v), {variant_name(c): t for c, t in _TUNE["timings"].get(k, {}).items()})
            for k, v in _TUNE["table"].items()}


_SITES = {1: "producer waits for a free stage", 2: "MMA waits for operands"}
_FAMILIES = {1: "conv", 4: "wgrad"}


def conv_timeouts(raise_error: bool = True):
    """Post-mortem of the conv kernels' bounded mbarrier waits (tc_utils.cuh): None, or a description of the first
    wait that timed out since the last call (the kernels drain instead of hanging / trapping; results are garbage)."""
    info = _C().conv_timeout_info()
    if not info[0]:
        return None
    site = int(info[1])
    msg = (f"conv pipeline timeout in the {_FAMILIES.get(site >> 4, '?')} kernel: "
           f"{_SITES.get(site & 15, 'site %d' % site)} (block {info[2]}, thread {info[3]}, parity {info[4]})")
    if raise_error:
        raise RuntimeError(msg)
    return msg


def _tuned(key, candidates, launch, accumulators=()):
    """Run ``launch(variant)`` with the best known variant for ``key``; time the candidates on first sight."""
    if _TUNE.get("force") is not None:                 # tools / tests: run exactly this variant
        return launch(_TUNE["force"])
    if not _TUNE["enabled"]:
        return launch(0)
    v = _TUNE["table"].get(key)
    if v is not None:
        return launch(v)
    if torch.cuda.is_current_stream_capturing() or len(candidates) < 2:
        return launch(0)                               # nothing to choose: the launcher's policy (and its tuning hooks)
    times = {}
    for c in candidates:
        try:
            launch(c)
            launch(c)
            a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            a.record()
            for _ in range(4):
                launch(c)
            b.record()
            b.synchronize()
            bad = conv_timeouts(raise_error=False)
            if bad is not None:                        # a variant that dead-locks on this shape is never chosen
                _TUNE.setdefault("rejected", {}).setdefault(key, {})[variant_name(c)] = bad
                continue
            times[c] = a.elapsed_time(b) / 4 * 1e3
        except RuntimeError:
            continue                                   # variant not applicable to this shape
    if not times:
        return launch(0)
    best = min(times, key=times.get)
    _TUNE["table"][key] = best
    _TUNE["timings"][key] = times
    for t in accumulators:                             # the trial launches accumulated BN statistics: start over
        t.zero_()
    return launch(best)


@functools.lru_cache(maxsize=None)
def sm_count(device_index: int = 0) -> int:
    return torch.cuda.get_device_properties(device_index).multi_processor_count


def _stream() -> int:
    return torch.cuda.current_stream().cuda_stream


def _ptr(t: Optional[torch.Tensor]) -> int:
    return 0 if t is None else t.data_ptr()


def _check_act(x: torch.Tensor, name: str = "x") -> None:
    if x.dtype != torch.bfloat16 or not x.is_cuda:
        raise TypeError(f"{name}: expected a CUDA bfloat16 tensor, got {x.dtype} on {x.device}")
    if x.dim() == 4 and not x.is_contiguous(memory_format=CL):
        raise ValueError(f"{name}: expected channels_last memory, strides={x.stride()}")
    if x.dim() == 2 and not x.is_contiguous():
        raise ValueError(f"{name}: expected a contiguous matrix")


class _ZeroRing:
    """Pre-zeroed fp32 scratch handed out in stream order.

    Every conv+BN unit needs a few hundred zeroed floats per step (BN sum / sum-of-squares accumulators, dgamma /
    dbeta scratch): ~110 `torch.zeros` launches per ResNet-50 step.  Slices of one arena are handed out
    sequentially instead and the arena is re-zeroed with ONE memset when it wraps.  Safe because every consumer of a
    slice is enqueued on the current stream right after its producer, i.e. before the wrap-around memset."""

    def __init__(self, device, numel: int = 1 << 21):
        self.buf = torch.zeros(numel, dtype=torch.float32, device=device)
        self.pos = 0

    def take(self, numel: int) -> torch.Tensor:
        n = (numel + 31) // 32 * 32                     # 128-byte granules
        if n > self.buf.numel():
            return torch.zeros(numel, dtype=torch.float32, device=self.buf.device)
        if self.pos + n > self.buf.numel():
            self.buf.zero_()
            self.pos = 0
        out = self.buf[self.pos:self.pos + numel]
        self.pos += n
        return out


_zero_rings = {}
_capture_ring = {"ring": None}


def begin_capture_scratch(device) -> None:
    """Call right after CUDA-graph capture of a step began (on the capture stream): the step's accumulators come
    from a dedicated arena whose memset is the first node of the graph, so every replay starts from zeros."""
    ring = _ZeroRing.__new__(_ZeroRing)
    ring.buf = torch.empty(1 << 21, dtype=torch.float32, device=device)
    ring.buf.zero_()                                   # captured memset
    ring.pos = 0
    ring.no_wrap = True
    _capture_ring["ring"] = ring


def end_capture_scratch() -> None:
    _capture_ring["ring"] = None


def zeros_f32(shape, device) -> torch.Tensor:
    """Zero-filled fp32 scratch for accumulators that are consumed on the current stream right away."""
    numel = 1
    for d in shape:
        numel *= int(d)
    cap = _capture_ring["ring"]
    if cap is not None:
        n = (numel + 31) // 32 * 32
        if cap.pos + n > cap.buf.numel():
            return torch.zeros(numel, dtype=torch.float32, device=device).view(*shape)     # captured memset node
        out = cap.buf[cap.pos:cap.pos + numel]
        cap.pos += n
        return out.view(*shape)
    key = (device.index or 0, torch.cuda.current_stream(device).cuda_stream)
    ring = _zero_rings.get(key)
    if ring is None:
        ring = _zero_rings[key] = _ZeroRing(device)
    return ring.take(numel).view(*shape)


def empty_act(n: int, c: int, h: int, w: int, device) -> torch.Tensor:
    return torch.empty((n, c, h, w), dtype=torch.bfloat16, device=device, memory_format=CL)


def _pad2(pad) -> Tuple[int, int]:
    """Padding as (pad_h, pad_w); an int means the same on both axes."""
    if isinstance(pad, (tuple, list)):
        return int(pad[0]), int(pad[1])
    return int(pad), int(pad)


def conv_out_hw(h: int, w: int, k: Tuple[int, int], stride: int, pad, dil: int = 1) -> Tuple[int, int]:
    ph, pw = _pad2(pad)
    return ((h + 2 * ph - dil * (k[0] - 1) - 1) // stride + 1, (w + 2 * pw - dil * (k[1] - 1) - 1) // stride + 1)


def _ceil_div(a: int, b: int) -> int:
    return -(-a // b)


# ------------------------------------------------------------------------------------------------
# stem geometry helpers (Cin <= 4): k-block = RPK filter rows x SP padded taps x 4 channels
# ------------------------------------------------------------------------------------------------
def stem_geometry(R: int, S: int) -> Tuple[int, int, int, int]:
    """Returns (SP, RPK, KB, RP): padded taps per row, rows per k-block, k-blocks, padded rows."""
    SP = 4 if S <= 4 else (8 if S <= 8 else 16)
    if S > 16:
        raise ValueError("stem kernels support at most 16 taps per filter row")
    RPK = 16 // SP
    KB = (R + RPK - 1) // RPK
    return SP, RPK, KB, KB * RPK


USE_STEM_TMA = os.environ.get("DDL_DISABLE_STEM_TMA", "0") != "1"
USE_TILE_TMA = os.environ.get("DDL_DISABLE_TILE_TMA", "0") != "1"
USE_TILE_S2 = os.environ.get("DDL_DISABLE_TILE_S2", "0") != "1"


@functools.lru_cache(maxsize=None)
def tile_geometry(P: int, Q: int, N: int, max_rows: int) -> Tuple[int, int, int]:
    """(tw, th, tn): the box of output pixels one TMA request covers (w fastest), tw*th*tn <= max_rows.

    The tensor core always multiplies ``max_rows`` rows, so the box is chosen to maximise the fraction of them that are
    real pixels over the whole tensor: fill of the box (tw*th*tn / max_rows) times the coverage overshoot of each axis.
    Full-width boxes with as many image rows as fit were the obvious choice, but for 14x14 maps that is 14x9 = 126 rows
    with the second box of every image more than half empty (77 % useful); 14x1x9 (one image row of nine consecutive
    images) is 96 % useful.  Ties prefer taller boxes (neighbouring taps of a 3x3 window re-read the same lines)."""
    if Q > max_rows:
        nw = -(-Q // max_rows)
        return -(-Q // nw), 1, 1
    best, best_key = (Q, 1, 1), None
    widths = sorted({Q} | {-(-Q // d) for d in (2, 3, 4) if Q // d >= 4})
    for tw in widths:
        cov_w = Q / (-(-Q // tw) * tw)
        for th in range(1, min(P, max_rows // tw) + 1):
            cov_h = P / (-(-P // th) * th)
            tns = [1] if th < P else list(range(1, min(N, max_rows // (tw * th)) + 1))
            if th < P:
                tns = list(range(1, min(N, max_rows // (tw * th)) + 1)) if th == 1 else [1]
            for tn in tns:
                rows = tw * th * tn
                if rows > max_rows:
                    continue
                cov_n = N / (-(-N // tn) * tn)
                eff = rows / max_rows * cov_w * cov_h * cov_n
                key = (round(eff, 4), th, tw)
                if best_key is None or key > best_key:
                    best, best_key = (tw, th, tn), key
    return best


def stem_tma_geometry(H: int, W: int, kernel: Tuple[int, int], stride: int, pad) -> Optional[Tuple[int, int, int]]:
    """(Hp, Wp, G) of the zero-padded, G-row-interleaved NHWC4 image the TMA-fed stem kernel reads (G = filter rows
    per k-block), or None when it does not apply: the per-output-column step of the tensor map (stride*G pixels of 8
    bytes) must be a multiple of 16 bytes."""
    if not USE_STEM_TMA or kernel[1] > 16:
        return None
    ph, pw = _pad2(pad)
    SP, RPK, KB, RP = stem_geometry(*kernel)
    if (stride * RPK) % 2 != 0:
        return None
    P, Q = conv_out_hw(H, W, kernel, stride, (ph, pw))
    Hp = max(H + 2 * ph, stride * (P - 1) + RPK * (KB - 1) + 1)
    Wp = max(W + 2 * pw, stride * (Q - 1) + SP)
    return Hp, Wp + (Wp % 2), RPK


def pad_image(x4: torch.Tensor, Hp: int, Wp: int, pt: int, pl: int, G: int = 1) -> torch.Tensor:
    """NHWC4 image -> zero-bordered [N, Hp, Wp, G, 4] copy with the source at (pt, pl); slot g of position (h, w)
    holds the pixel of row h + g (the 128 bytes one stem k-block needs become contiguous)."""
    _check_act(x4)
    N, c, H, W = x4.shape
    if c != 4:
        raise ValueError("pad_image expects an NHWC4 tensor")
    out = torch.empty((N, Hp, Wp, G, 4), dtype=torch.bfloat16, device=x4.device)
    _C().pad_nhwc4(x4.data_ptr(), out.data_ptr(), N, H, W, Hp, Wp, pt, pl, G, _stream())
    return out


def stem_prepare(x4: torch.Tensor, kernel: Tuple[int, int], stride: int, pad, dil: int = 1) -> Optional[torch.Tensor]:
    """The zero-padded, row-interleaved copy of an NHWC4 image batch that the TMA-fed stem kernels read, or None when
    that path does not apply.  Forward and weight-gradient kernels of the same layer can share it (``prepadded=``)."""
    if x4.shape[1] != 4 or dil != 1:
        return None
    ph, pw = _pad2(pad)
    geo = stem_tma_geometry(x4.shape[2], x4.shape[3], kernel, stride, (ph, pw))
    if geo is None:
        return None
    return pad_image(x4, geo[0], geo[1], ph, pw, geo[2])


def supports_conv(cin: int, cout: int) -> bool:
    """Shapes the wgmma implicit-GEMM kernels handle natively: channel counts that are multiples of 8 (one 16-byte
    vector; partial 64-channel k-blocks / N tiles are zero-filled or masked in the kernels) or an NHWC4 stem."""
    return cout % 8 == 0 and (cin % 8 == 0 or cin <= 4)


def supports_grouped(cin: int, cout: int, groups: int) -> bool:
    """The whole-groups-per-tile subset of the grouped convolutions: ``cin == cout``, a multiple of 64, split into groups
    whose width divides 64 (a 64-channel tile then holds whole groups) and is a multiple of 4 (each 16-byte
    weight-gradient vector lies in one group).  :func:`grouped_conv_native` is what the kernels take."""
    if groups <= 1:
        return supports_conv(cin, cout)
    if cin != cout or cin % groups != 0 or cin % 64 != 0:
        return False
    cg = cin // groups
    return 64 % cg == 0 and cg % 4 == 0


def grouped_conv_native(cin: int, cout: int, groups: int) -> bool:
    """Grouped convolutions (``groups`` > 1) the conv kernels run natively: :func:`supports_grouped`, or ``cin == cout``
    a multiple of 8 in groups of a width ``cg`` that is a multiple of 8 (group bundles, :func:`grouped_bundle`).
    Depthwise convolutions (``cg == 1``) are not among them; other shapes take the composite path."""
    if groups <= 1:
        return False
    if supports_grouped(cin, cout, groups):
        return True
    return cin == cout and cin % groups == 0 and cin % 8 == 0 and (cin // groups) % 8 == 0


def grouped_bundle(cg: int) -> Tuple[int, int]:
    """(Wb, T) of the grouped kernels for group width ``cg``: a bundle is ``max(1, 64 // cg)`` consecutive groups, Wb
    channels wide, and spans T = ceil(Wb / 64) N tiles of 64 channels and T k-blocks of 64 channels per filter tap."""
    wb = max(1, 64 // cg) * cg
    return wb, _ceil_div(wb, 64)


def grouped_expanded_shape(c: int, taps: int, groups: int) -> Tuple[int, int]:
    """Shape [nbundles * T * 64, taps * T * 64] of :func:`expand_grouped_weight`'s result."""
    wb, t = grouped_bundle(c // groups)
    return _ceil_div(c, wb) * t * 64, taps * t * 64


def _depthwise_ok(k_want: int, c: int, kernel, stride: int, pad, dil: int, groups: int) -> bool:
    k = (kernel, kernel) if isinstance(kernel, int) else tuple(kernel)
    return (groups == c and c > 0 and c % 8 == 0 and k == (k_want, k_want) and stride in (1, 2)
            and _pad2(pad) == (k_want // 2, k_want // 2) and dil == 1)


def supports_depthwise(c: int, kernel, stride: int, pad, dil: int, groups: int) -> bool:
    """Depthwise convolutions the 3x3 stencil kernels of csrc/ops/depthwise.cu handle: ``groups == Cin == Cout = c``
    with ``c % 8 == 0``, a 3x3 kernel, stride 1 or 2, padding 1 and dilation 1 (MobileNetV2's depthwise layers and
    MobileNetV3's 3x3 ones).  The 5x5 kernels have their own predicate, :func:`supports_depthwise5`."""
    return _depthwise_ok(3, c, kernel, stride, pad, dil, groups)


def supports_depthwise5(c: int, kernel, stride: int, pad, dil: int, groups: int) -> bool:
    """Depthwise convolutions the 5x5 stencil kernels of csrc/ops/depthwise5.cu handle: ``groups == Cin == Cout = c``
    with ``c % 8 == 0``, a 5x5 kernel, stride 1 or 2, padding 2 and dilation 1 (MobileNetV3's 5x5 layers)."""
    return _depthwise_ok(5, c, kernel, stride, pad, dil, groups)


def depthwise_native(c: int, kernel, stride: int, pad, dil: int, groups: int) -> bool:
    """Whether one of the native depthwise kernel families (3x3 or 5x5) takes this convolution."""
    return supports_depthwise(c, kernel, stride, pad, dil, groups) or \
        supports_depthwise5(c, kernel, stride, pad, dil, groups)


def supports_depthwise7(c: int, kernel, stride: int, pad, dil: int, groups: int) -> bool:
    """Depthwise convolutions the 7x7 kernels of csrc/ops/depthwise7.cu handle: ``groups == Cin == Cout = c`` with
    ``c % 8 == 0``, a 7x7 kernel, stride 1, padding 3 and dilation 1 (ConvNeXt's depthwise layers, which carry a bias).
    They are separate from :func:`depthwise_native`, which decides what ``conv_bn_act`` sends to its depthwise node."""
    return _depthwise_ok(7, c, kernel, stride, pad, dil, groups) and stride == 1


def _check_dw(c: int, w_bf16: torch.Tensor, stride: int, k: int) -> None:
    if not depthwise_native(c, (k, k), stride, k // 2, 1, c):
        raise ValueError(f"depthwise {k}x{k} conv with {c} channels, stride {stride} is not supported by the native "
                         "kernels")
    if w_bf16.dtype != torch.bfloat16 or w_bf16.numel() != c * k * k or not w_bf16.is_contiguous() \
            or w_bf16.device.type != "cuda":
        raise ValueError(f"depthwise conv: expected contiguous CUDA bf16 weights [C, {k * k}] (KRSC of [C, 1, {k}, {k}])")


def _check_aligned(t: torch.Tensor, name: str) -> None:
    if t.data_ptr() % 16 != 0:
        raise ValueError(f"{name}: the depthwise kernels need 16-byte aligned activations")


def dwconv_fwd(x: torch.Tensor, w_bf16: torch.Tensor, stride: int, stats: bool = False, k: int = 3):
    """Depthwise k x k convolution (k = 3 with padding 1 or k = 5 with padding 2): y[n, c] = conv(x[n, c], w[c]).
    ``w_bf16``: [C, k*k] bf16.  With ``stats`` also the per-channel (sum, sumsq) of the bf16 y as fp32 [2, C] (same
    contract as ``conv_fwd(stats=True)``)."""
    _check_act(x)
    N, Ch, H, W = x.shape
    _check_dw(Ch, w_bf16, stride, k)
    _check_aligned(x, "x")
    P, Q = conv_out_hw(H, W, (k, k), stride, k // 2)
    y = empty_act(N, Ch, P, Q, x.device)
    st = zeros_f32((2, Ch), x.device) if stats else None
    _C().dwconv_fwd(x.data_ptr(), w_bf16.data_ptr(), y.data_ptr(), st[0].data_ptr() if stats else 0,
                    st[1].data_ptr() if stats else 0, N, H, W, Ch, P, Q, stride, sm_count(x.device.index or 0), _stream(),
                    k)
    return (y, st) if stats else y


def dwconv_dgrad(dy: torch.Tensor, w_bf16: torch.Tensor, x_shape, stride: int, k: int = 3) -> torch.Tensor:
    """dx = conv_transpose(dy, w) of :func:`dwconv_fwd` (every element written once)."""
    _check_act(dy, "dy")
    N, Ch, H, W = x_shape
    _check_dw(Ch, w_bf16, stride, k)
    _check_aligned(dy, "dy")
    P, Q = conv_out_hw(H, W, (k, k), stride, k // 2)
    if tuple(dy.shape) != (N, Ch, P, Q):
        raise ValueError(f"dwconv_dgrad: dy has shape {tuple(dy.shape)}, expected {(N, Ch, P, Q)}")
    dx = empty_act(N, Ch, H, W, dy.device)
    _C().dwconv_dgrad(dy.data_ptr(), w_bf16.data_ptr(), dx.data_ptr(), N, H, W, Ch, P, Q, stride,
                      sm_count(dy.device.index or 0), _stream(), k)
    return dx


def dwconv_wgrad(x: torch.Tensor, dy: torch.Tensor, grad_w: torch.Tensor, stride: int, k: int = 3) -> None:
    """grad_w[C][k][k] (fp32, KRSC of [C, 1, k, k]) += the weight gradient of :func:`dwconv_fwd`."""
    _check_act(x)
    _check_act(dy, "dy")
    N, Ch, H, W = x.shape
    if not depthwise_native(Ch, (k, k), stride, k // 2, 1, Ch):
        raise ValueError(f"depthwise {k}x{k} conv with {Ch} channels, stride {stride} is not supported by the native "
                         "kernels")
    _check_aligned(x, "x")
    _check_aligned(dy, "dy")
    P, Q = conv_out_hw(H, W, (k, k), stride, k // 2)
    if tuple(dy.shape) != (N, Ch, P, Q):
        raise ValueError(f"dwconv_wgrad: dy has shape {tuple(dy.shape)}, expected {(N, Ch, P, Q)}")
    if grad_w.dtype != torch.float32 or grad_w.numel() != Ch * k * k or not grad_w.is_contiguous(memory_format=CL) \
            or not grad_w.is_cuda:
        raise ValueError(f"dwconv_wgrad: grad_w must be a CUDA fp32 [C, 1, {k}, {k}] (KRSC) tensor")
    _C().dwconv_wgrad(x.data_ptr(), dy.data_ptr(), grad_w.data_ptr(), N, H, W, Ch, P, Q, stride,
                      sm_count(x.device.index or 0), _stream(), k)


# ------------------------------------------------------------------------------------------------
# depthwise 7x7 with a bias (csrc/ops/depthwise7.cu) and the ConvNeXt row kernels (csrc/ops/convnext.cu)
# ------------------------------------------------------------------------------------------------
def _check_dw7(x: torch.Tensor, name: str, w_bf16: Optional[torch.Tensor] = None) -> None:
    _check_act(x, name)
    if x.dim() != 4 or not supports_depthwise7(x.shape[1], (7, 7), 1, 3, 1, x.shape[1]):
        raise ValueError(f"{name}: the depthwise 7x7 kernels need a 4-D activation with a multiple of 8 channels")
    _check_aligned(x, name)
    if w_bf16 is not None and (w_bf16.dtype != torch.bfloat16 or w_bf16.numel() != x.shape[1] * 49
                               or not w_bf16.is_contiguous() or not w_bf16.is_cuda):
        raise ValueError("depthwise 7x7: expected contiguous CUDA bf16 weights [C, 49] (KRSC of [C, 1, 7, 7])")


def _check_f32_vec(t: Optional[torch.Tensor], n: int, name: str) -> None:
    if t is not None and (t.dtype != torch.float32 or not t.is_cuda or t.numel() != n or not t.is_contiguous()):
        raise ValueError(f"{name}: expected a contiguous CUDA fp32 tensor of {n} elements")


def dwconv7_fwd(x: torch.Tensor, w_bf16: torch.Tensor, bias: torch.Tensor, l1: bool = False) -> torch.Tensor:
    """y = depthwise 7x7 conv (stride 1, padding 3) of x with the bf16 weights [C, 49], plus the fp32 bias [C].
    ``l1``: run the L1 mapping of the 5x5 kernels instead of the shared-memory halo tile (tools/depthwise_bench.py times
    the two against each other; the model path uses the halo tile)."""
    _check_dw7(x, "x", w_bf16)
    N, Ch, H, W = x.shape
    _check_f32_vec(bias, Ch, "bias")
    y = torch.empty_like(x)
    _C().dwconv7_fwd(x.data_ptr(), w_bf16.data_ptr(), bias.data_ptr(), y.data_ptr(), N, H, W, Ch,
                     sm_count(x.device.index or 0), _stream(), int(l1))
    return y


def dwconv7_dgrad(dy: torch.Tensor, w_bf16: torch.Tensor, add: Optional[torch.Tensor] = None,
                  l1: bool = False) -> torch.Tensor:
    """dx = conv_transpose(dy, w) of :func:`dwconv7_fwd` (+ ``add``, a same-shape tensor added in the store); ``l1`` as
    in :func:`dwconv7_fwd`."""
    _check_dw7(dy, "dy", w_bf16)
    if add is not None:
        _check_act(add, "add")
        _check_aligned(add, "add")
        if add.shape != dy.shape:
            raise ValueError("dwconv7_dgrad: add must have the shape of dy")
    N, Ch, H, W = dy.shape
    dx = torch.empty_like(dy)
    _C().dwconv7_dgrad(dy.data_ptr(), w_bf16.data_ptr(), _ptr(add), dx.data_ptr(), N, H, W, Ch,
                       sm_count(dy.device.index or 0), _stream(), int(l1))
    return dx


def dwconv7_wgrad(x: torch.Tensor, dy: torch.Tensor, grad_w: torch.Tensor, grad_b: Optional[torch.Tensor]) -> None:
    """grad_w [C, 1, 7, 7] (fp32 KRSC) += the weight gradient of :func:`dwconv7_fwd`; grad_b [C] += sum of dy."""
    _check_dw7(x, "x")
    _check_dw7(dy, "dy")
    if dy.shape != x.shape:
        raise ValueError("dwconv7_wgrad: dy must have the shape of x")
    N, Ch, H, W = x.shape
    if grad_w.dtype != torch.float32 or grad_w.numel() != Ch * 49 or not grad_w.is_contiguous(memory_format=CL) \
            or not grad_w.is_cuda:
        raise ValueError("dwconv7_wgrad: grad_w must be a CUDA fp32 [C, 1, 7, 7] (KRSC) tensor")
    _check_f32_vec(grad_b, Ch, "grad_b")
    _C().dwconv7_wgrad(x.data_ptr(), dy.data_ptr(), grad_w.data_ptr(), _ptr(grad_b), N, H, W, Ch,
                       sm_count(x.device.index or 0), _stream())


def supports_layer_norm(c: int) -> bool:
    """Channel counts the LayerNorm kernels take: C % 8 == 0 with C / 8 = T * V, T the largest power of two <= 32
    dividing C / 8 and V <= 6 (every ConvNeXt width, 96 to 1536)."""
    if c <= 0 or c % 8 != 0:
        return False
    v = c // 8
    t = 1
    while t < 32 and v % (2 * t) == 0:
        t *= 2
    return v // t <= 6


def _rows(x: torch.Tensor) -> Tuple[int, int]:
    """(rows, channels) of an NHWC activation [N, C, H, W] or a matrix [N, C]."""
    if x.dim() == 4:
        return x.shape[0] * x.shape[2] * x.shape[3], x.shape[1]
    if x.dim() == 2:
        return x.shape[0], x.shape[1]
    raise ValueError("expected an NHWC activation [N, C, H, W] or a matrix [N, C]")


def layer_norm_fwd(x: torch.Tensor, gamma: torch.Tensor, beta: torch.Tensor, eps: float):
    """LayerNorm over the channels of every row: returns (y bf16 like x, mean fp32 [rows], rstd fp32 [rows])."""
    _check_act(x)
    _check_aligned(x, "x")
    M, Ch = _rows(x)
    if not supports_layer_norm(Ch):
        raise ValueError(f"layer_norm: {Ch} channels are not supported by the native kernels")
    _check_f32_vec(gamma, Ch, "gamma")
    _check_f32_vec(beta, Ch, "beta")
    y = torch.empty_like(x)
    mean = torch.empty(M, dtype=torch.float32, device=x.device)
    rstd = torch.empty(M, dtype=torch.float32, device=x.device)
    _C().layer_norm_fwd(x.data_ptr(), gamma.data_ptr(), beta.data_ptr(), y.data_ptr(), mean.data_ptr(), rstd.data_ptr(),
                        M, Ch, float(eps), sm_count(x.device.index or 0), _stream())
    return y, mean, rstd


def layer_norm_bwd(dy: torch.Tensor, x: torch.Tensor, mean: torch.Tensor, rstd: torch.Tensor, gamma: torch.Tensor,
                   grad_gamma: Optional[torch.Tensor], grad_beta: Optional[torch.Tensor]) -> torch.Tensor:
    """dx of :func:`layer_norm_fwd` from the saved x, mean and rstd; grad_gamma += sum dy * xhat, grad_beta += sum dy."""
    _check_act(dy, "dy")
    _check_act(x)
    _check_aligned(dy, "dy")
    if dy.shape != x.shape:
        raise ValueError("layer_norm_bwd: dy must have the shape of x")
    M, Ch = _rows(x)
    for t, name in ((gamma, "gamma"), (grad_gamma, "grad_gamma"), (grad_beta, "grad_beta")):
        _check_f32_vec(t, Ch, name)
    dx = torch.empty_like(x)
    _C().layer_norm_bwd(dy.data_ptr(), x.data_ptr(), mean.data_ptr(), rstd.data_ptr(), gamma.data_ptr(), dx.data_ptr(),
                        _ptr(grad_gamma), _ptr(grad_beta), M, Ch, sm_count(x.device.index or 0), _stream())
    return dx


def gelu_fwd(h: torch.Tensor) -> torch.Tensor:
    """g = h * Phi(h) (exact GELU) elementwise."""
    _check_act(h, "h")           # dense NHWC or a contiguous matrix: elementwise over the memory
    if h.numel() % 8 != 0:
        raise ValueError("gelu_fwd: expected a multiple of 8 elements")
    _check_aligned(h, "h")
    g = torch.empty_like(h)
    _C().gelu_fwd(h.data_ptr(), g.data_ptr(), h.numel(), sm_count(h.device.index or 0), _stream())
    return g


def gelu_bwd(dg: torch.Tensor, h: torch.Tensor, grad_bias: Optional[torch.Tensor]) -> torch.Tensor:
    """dh = dg * (Phi(h) + h phi(h)) from the saved pre-activation h; grad_bias [C] += the column sums of dh."""
    _check_act(dg, "dg")
    _check_act(h, "h")
    if dg.shape != h.shape:
        raise ValueError("gelu_bwd: dg must have the shape of h")
    M, Ch = _rows(h)
    if Ch % 8 != 0 or Ch > 8192:
        raise ValueError("gelu_bwd: the channel count must be a multiple of 8, at most 8192")
    _check_aligned(dg, "dg")
    _check_aligned(h, "h")
    _check_f32_vec(grad_bias, Ch, "grad_bias")
    dh = torch.empty_like(h)
    _C().gelu_bwd(dg.data_ptr(), h.data_ptr(), dh.data_ptr(), _ptr(grad_bias), M, Ch, sm_count(h.device.index or 0),
                  _stream())
    return dh


def _check_keep(keep: Optional[torch.Tensor], n: int) -> None:
    if keep is not None and (keep.dtype != torch.float32 or not keep.is_cuda or keep.dim() != 1 or keep.shape[0] != n
                             or not keep.is_contiguous()):
        raise ValueError(f"layer scale: keep must be a contiguous CUDA fp32 [{n}] tensor")


def layer_scale_fwd(y: torch.Tensor, ls: torch.Tensor, keep: Optional[torch.Tensor], x: torch.Tensor) -> torch.Tensor:
    """z = ls[c] * y * keep[n] + x for NHWC activations y, x [N, C, H, W] (``keep``: stochastic depth, or None)."""
    _check_act(y, "y")
    _check_act(x)
    if y.dim() != 4 or y.shape != x.shape or y.shape[1] % 8 != 0:
        raise ValueError("layer_scale_fwd: y and x must be NHWC activations of one shape, C a multiple of 8")
    _check_aligned(y, "y")
    _check_aligned(x, "x")
    N, Ch, H, W = y.shape
    _check_f32_vec(ls, Ch, "ls")
    _check_keep(keep, N)
    z = torch.empty_like(x)
    _C().layer_scale_fwd(y.data_ptr(), ls.data_ptr(), _ptr(keep), x.data_ptr(), z.data_ptr(), N * H * W, Ch, H * W,
                         sm_count(y.device.index or 0), _stream())
    return z


def layer_scale_bwd(dz: torch.Tensor, y: torch.Tensor, ls: torch.Tensor, keep: Optional[torch.Tensor],
                    grad_ls: Optional[torch.Tensor], grad_bias: Optional[torch.Tensor]) -> torch.Tensor:
    """dy = dz * ls[c] * keep[n]; grad_ls += sum dz * keep * y; grad_bias (fc2's) += sum dy."""
    _check_act(dz, "dz")
    _check_act(y, "y")
    if dz.shape != y.shape or y.dim() != 4:
        raise ValueError("layer_scale_bwd: dz must have the shape of y")
    _check_aligned(dz, "dz")
    _check_aligned(y, "y")
    N, Ch, H, W = y.shape
    if Ch % 8 != 0 or Ch > 4096:
        raise ValueError("layer_scale_bwd: the channel count must be a multiple of 8, at most 4096")
    for t, name in ((ls, "ls"), (grad_ls, "grad_ls"), (grad_bias, "grad_bias")):
        _check_f32_vec(t, Ch, name)
    _check_keep(keep, N)
    dy = torch.empty_like(y)
    _C().layer_scale_bwd(dz.data_ptr(), y.data_ptr(), ls.data_ptr(), _ptr(keep), dy.data_ptr(), _ptr(grad_ls),
                         _ptr(grad_bias), N * H * W, Ch, H * W, sm_count(y.device.index or 0), _stream())
    return dy


# ------------------------------------------------------------------------------------------------
# ViT: multi-head self-attention (csrc/ops/attention.cu) and the token-row kernels (csrc/ops/vit.cu)
# ------------------------------------------------------------------------------------------------
def supports_attention(L: int, heads: int, head_dim: int) -> bool:
    """Shapes the attention kernels take: head dim 64 and C = 64 * heads (any L >= 1)."""
    return head_dim == 64 and 0 < heads <= 65535 and L >= 1


def _check_rows(t: torch.Tensor, rows: int, cols: int, name: str) -> None:
    if t.dtype != torch.bfloat16 or not t.is_cuda or t.dim() != 2 or tuple(t.shape) != (rows, cols) \
            or not t.is_contiguous():
        raise ValueError(f"{name}: expected a contiguous CUDA bf16 [{rows}, {cols}] matrix, got {t.dtype} "
                         f"{tuple(t.shape)} on {t.device}")
    _check_aligned(t, name)


def _attn_dims(qkv: torch.Tensor, num_heads: int, L: int) -> Tuple[int, int]:
    if qkv.dim() != 2 or qkv.shape[1] % 3 != 0 or L <= 0 or qkv.shape[0] % L != 0:
        raise ValueError("attention: qkv must be [N*L, 3C]")
    C = qkv.shape[1] // 3
    if C % num_heads != 0 or not supports_attention(L, num_heads, C // num_heads):
        raise ValueError(f"attention: head dim {C // max(num_heads, 1)} is not supported by the native kernels (64 only)")
    return qkv.shape[0] // L, C


def attention_fwd(qkv: torch.Tensor, num_heads: int, L: int):
    """O [N*L, C] = softmax(Q K^T / sqrt(64)) V per (image, head) from the packed in-projection output qkv [N*L, 3C];
    returns (O, lse fp32 [N, H, L])."""
    N, C = _attn_dims(qkv, num_heads, L)
    _check_rows(qkv, N * L, 3 * C, "qkv")
    o = torch.empty((N * L, C), dtype=torch.bfloat16, device=qkv.device)
    lse = torch.empty((N, num_heads, L), dtype=torch.float32, device=qkv.device)
    _C().attention_fwd(qkv.data_ptr(), o.data_ptr(), lse.data_ptr(), N, L, num_heads, C, _stream())
    return o, lse


def attention_bwd(dout: torch.Tensor, qkv: torch.Tensor, o: torch.Tensor, lse: torch.Tensor, num_heads: int,
                  L: int) -> torch.Tensor:
    """dqkv [N*L, 3C] (qkv's layout) of :func:`attention_fwd` from dO and the saved qkv, O and lse."""
    N, C = _attn_dims(qkv, num_heads, L)
    _check_rows(qkv, N * L, 3 * C, "qkv")
    _check_rows(o, N * L, C, "o")
    _check_rows(dout, N * L, C, "dout")
    if lse.dtype != torch.float32 or tuple(lse.shape) != (N, num_heads, L) or not lse.is_contiguous():
        raise ValueError("attention_bwd: lse must be the contiguous fp32 [N, H, L] of the forward")
    dqkv = torch.empty_like(qkv)
    delta = torch.empty((N, num_heads, L), dtype=torch.float32, device=qkv.device)
    _C().attention_bwd(qkv.data_ptr(), o.data_ptr(), dout.data_ptr(), lse.data_ptr(), delta.data_ptr(),
                       dqkv.data_ptr(), N, L, num_heads, C, _stream())
    return dqkv


def add_layer_norm_fwd(x: torch.Tensor, a: torch.Tensor, gamma: torch.Tensor, beta: torch.Tensor, eps: float):
    """x1 = x + a and t = LayerNorm(x1) over the rows of [M, C] matrices: returns (x1, t, mean fp32 [M], rstd fp32 [M])."""
    M, Ch = _rows(x)
    _check_rows(x, M, Ch, "x")
    _check_rows(a, M, Ch, "a")
    if x.dim() != 2 or not supports_layer_norm(Ch):
        raise ValueError(f"add_layer_norm: {Ch} channels are not supported by the native kernels")
    _check_f32_vec(gamma, Ch, "gamma")
    _check_f32_vec(beta, Ch, "beta")
    x1, t = torch.empty_like(x), torch.empty_like(x)
    mean = torch.empty(M, dtype=torch.float32, device=x.device)
    rstd = torch.empty(M, dtype=torch.float32, device=x.device)
    _C().add_layer_norm_fwd(x.data_ptr(), a.data_ptr(), gamma.data_ptr(), beta.data_ptr(), x1.data_ptr(), t.data_ptr(),
                            mean.data_ptr(), rstd.data_ptr(), M, Ch, float(eps), sm_count(x.device.index or 0), _stream())
    return x1, t, mean, rstd


def layer_norm_bwd_add(dy: torch.Tensor, x: torch.Tensor, mean: torch.Tensor, rstd: torch.Tensor, gamma: torch.Tensor,
                       dres: torch.Tensor, grad_gamma: Optional[torch.Tensor],
                       grad_beta: Optional[torch.Tensor]) -> torch.Tensor:
    """dx = :func:`layer_norm_bwd` (dy) + dres over [M, C] rows, with the same grad_gamma / grad_beta sums."""
    M, Ch = _rows(x)
    for t, name in ((dy, "dy"), (x, "x"), (dres, "dres")):
        _check_rows(t, M, Ch, name)
    if not supports_layer_norm(Ch):
        raise ValueError(f"layer_norm_bwd_add: {Ch} channels are not supported by the native kernels")
    _check_f32_vec(mean, M, "mean")
    _check_f32_vec(rstd, M, "rstd")
    for t, name in ((gamma, "gamma"), (grad_gamma, "grad_gamma"), (grad_beta, "grad_beta")):
        _check_f32_vec(t, Ch, name)
    dx = torch.empty_like(x)
    _C().layer_norm_bwd_add(dy.data_ptr(), x.data_ptr(), mean.data_ptr(), rstd.data_ptr(), gamma.data_ptr(),
                            dres.data_ptr(), dx.data_ptr(), _ptr(grad_gamma), _ptr(grad_beta), M, Ch,
                            sm_count(x.device.index or 0), _stream())
    return dx


def patchify(img: torch.Tensor, patch: int) -> torch.Tensor:
    """NHWC4 image [N, 4, H, W] -> patch rows [N * (H/P) * (W/P), P*P*3] in (r, s, c) order: the GEMM operand of a
    channels_last conv_proj weight [C, 3, P, P] taken as the [C, 3*P*P] matrix it is in memory."""
    _check_act(img, "img")
    N, c4, H, W = img.shape
    if img.dim() != 4 or c4 != 4 or H % patch != 0 or W % patch != 0:
        raise ValueError(f"patchify: expected an NHWC4 image whose sides are multiples of {patch}")
    rows = N * (H // patch) * (W // patch)
    out = torch.empty((rows, 3 * patch * patch), dtype=torch.bfloat16, device=img.device)
    _C().patchify(img.data_ptr(), out.data_ptr(), N, H, W, patch, sm_count(img.device.index or 0), _stream())
    return out


def tokens_fwd(patch_rows: torch.Tensor, cls: torch.Tensor, pos: torch.Tensor, N: int) -> torch.Tensor:
    """tokens [N*L, C]: row (n, 0) = cls + pos[0], row (n, 1+p) = patch_rows[n*(L-1) + p] + pos[1+p] (cls [C] and
    pos [L, C] fp32)."""
    C = cls.numel()
    L = pos.numel() // max(C, 1)
    if C % 8 != 0 or L < 2 or pos.numel() != L * C:
        raise ValueError("tokens_fwd: pos must hold L >= 2 rows of C (a multiple of 8) columns")
    _check_rows(patch_rows, N * (L - 1), C, "patch_rows")
    _check_f32_vec(cls, C, "cls")
    _check_f32_vec(pos, L * C, "pos")
    tok = torch.empty((N * L, C), dtype=torch.bfloat16, device=patch_rows.device)
    _C().tokens_fwd(patch_rows.data_ptr(), cls.data_ptr(), pos.data_ptr(), tok.data_ptr(), N, L, C,
                    sm_count(tok.device.index or 0), _stream())
    return tok


def tokens_bwd(dtok: torch.Tensor, N: int, L: int, grad_pos: Optional[torch.Tensor], grad_cls: Optional[torch.Tensor],
               grad_bias: Optional[torch.Tensor], want_dpatch: bool = True) -> Optional[torch.Tensor]:
    """Backward of :func:`tokens_fwd`: returns dpatch [N*(L-1), C] (the patch rows of dtok, or None); grad_pos [L, C] +=
    sum over images, grad_cls [C] += that of token 0, grad_bias [C] += sum over the patch tokens (each optional)."""
    C = dtok.shape[1]
    if L < 2 or C % 8 != 0:
        raise ValueError("tokens_bwd: L >= 2 and C a multiple of 8")
    _check_rows(dtok, N * L, C, "dtok")
    _check_f32_vec(grad_pos, L * C, "grad_pos")
    _check_f32_vec(grad_cls, C, "grad_cls")
    _check_f32_vec(grad_bias, C, "grad_bias")
    dpatch = torch.empty((N * (L - 1), C), dtype=torch.bfloat16, device=dtok.device) if want_dpatch else None
    colsum = torch.empty((L, C), dtype=torch.float32, device=dtok.device)
    _C().tokens_bwd(dtok.data_ptr(), _ptr(dpatch), colsum.data_ptr(), _ptr(grad_pos), _ptr(grad_cls), _ptr(grad_bias),
                    N, L, C, _stream())
    return dpatch


# ------------------------------------------------------------------------------------------------
# Swin: shifted-window attention (csrc/ops/window_attention.cu) and patch merging (csrc/ops/swin.cu)
# ------------------------------------------------------------------------------------------------
def supports_window_attention(H: int, W: int, window: int, heads: int, head_dim: int) -> bool:
    """Shapes the window-attention kernels take: window 7, head dim 32, H and W multiples of 7 (no padding)."""
    return (window == 7 and head_dim == 32 and 0 < heads <= 65535 and H > 0 and W > 0 and H % 7 == 0 and W % 7 == 0
            and (H // 7) * (W // 7) <= 65535)


def supports_patch_merge(H: int, W: int, C: int) -> bool:
    """Maps the patch-merging kernels take: H and W even, C a multiple of 8 up to 512 (LayerNorm over 4C <= 2048)."""
    return H > 0 and W > 0 and H % 2 == 0 and W % 2 == 0 and 8 <= C <= 512 and C % 8 == 0


def window_shift(H: int, W: int, window: int, shift: int) -> Tuple[int, int]:
    """torchvision's per-side shift: 0 on a side whose (padded) size is at most the window."""
    ph, pw = -(-H // window) * window, -(-W // window) * window
    return (0 if ph <= window else shift), (0 if pw <= window else shift)


def _win_check(qkv: torch.Tensor, table: torch.Tensor, heads: int, N: int, H: int, W: int, shift: int):
    C = qkv.shape[1] // 3 if qkv.dim() == 2 else 0
    if C == 0 or C % heads != 0 or not supports_window_attention(H, W, 7, heads, C // heads):
        raise ValueError(f"window_attention: H={H}, W={W}, {heads} heads of {C // max(heads, 1)} are not supported by the "
                         "native kernels (window 7, head dim 32, H and W multiples of 7)")
    if not 0 <= shift < 7:
        raise ValueError("window_attention: shift must be in [0, 7)")
    _check_rows(qkv, N * H * W, 3 * C, "qkv")
    if table.dtype != torch.float32 or tuple(table.shape) != (169, heads) or not table.is_contiguous():
        raise ValueError(f"window_attention: table must be the contiguous fp32 [169, {heads}] parameter")
    return C


def window_attention_fwd(qkv: torch.Tensor, table: torch.Tensor, heads: int, N: int, H: int, W: int, shift: int):
    """Shifted-window attention (window 7, head dim 32) on the image-order qkv rows [N*H*W, 3C] with the relative-position
    bias ``table`` [169, heads] fp32: returns (O [N*H*W, C] in image order, lse fp32 [N*H*W, heads])."""
    C = _win_check(qkv, table, heads, N, H, W, shift)
    sy, sx = window_shift(H, W, 7, shift)
    o = torch.empty((N * H * W, C), dtype=torch.bfloat16, device=qkv.device)
    lse = torch.empty((N * H * W, heads), dtype=torch.float32, device=qkv.device)
    _C().window_attention_fwd(qkv.data_ptr(), table.data_ptr(), o.data_ptr(), lse.data_ptr(), N, H, W, heads, C, sy, sx,
                              _stream())
    return o, lse


def window_attention_bwd(dout: torch.Tensor, qkv: torch.Tensor, table: torch.Tensor, o: torch.Tensor, lse: torch.Tensor,
                         heads: int, N: int, H: int, W: int, shift: int,
                         grad_table: Optional[torch.Tensor]) -> torch.Tensor:
    """dqkv [N*H*W, 3C] (qkv's layout) of :func:`window_attention_fwd`; grad_table [169, heads] += the bias gradient
    (optional).  Deterministic: no atomics."""
    C = _win_check(qkv, table, heads, N, H, W, shift)
    sy, sx = window_shift(H, W, 7, shift)
    _check_rows(o, N * H * W, C, "o")
    _check_rows(dout, N * H * W, C, "dout")
    if lse.dtype != torch.float32 or tuple(lse.shape) != (N * H * W, heads) or not lse.is_contiguous():
        raise ValueError("window_attention_bwd: lse must be the contiguous fp32 [N*H*W, heads] of the forward")
    if grad_table is not None and (grad_table.dtype != torch.float32 or tuple(grad_table.shape) != (169, heads)
                                   or not grad_table.is_contiguous()):
        raise ValueError("window_attention_bwd: grad_table must be a contiguous fp32 [169, heads] buffer")
    dqkv = torch.empty_like(qkv)
    scratch = torch.empty(_C().window_attention_bwd_scratch_floats(N, H, heads), dtype=torch.float32,
                          device=qkv.device)
    _C().window_attention_bwd(qkv.data_ptr(), table.data_ptr(), o.data_ptr(), dout.data_ptr(), lse.data_ptr(),
                              dqkv.data_ptr(), _ptr(grad_table), scratch.data_ptr(), N, H, W, heads, C, sy, sx,
                              _stream())
    return dqkv


# ------------------------------------------------------------------------------------------------
# MaxViT: grid / window partition attention (csrc/ops/window_attention.cu)
# ------------------------------------------------------------------------------------------------
def supports_grid_attention(H: int, W: int, partition: int, heads: int, head_dim: int) -> bool:
    """Shapes the partition-attention kernels take: partition 7, head dim 32, a square map H = W, a multiple of 7."""
    return (partition == 7 and head_dim == 32 and 0 < heads <= 65535 and H > 0 and H == W and H % 7 == 0
            and (H // 7) ** 2 <= 65535)


def _grid_check(qkv: torch.Tensor, table: torch.Tensor, heads: int, N: int, H: int, W: int):
    C = qkv.shape[1] // 3 if qkv.dim() == 2 else 0
    if C == 0 or C % heads != 0 or not supports_grid_attention(H, W, 7, heads, C // heads):
        raise ValueError(f"grid_attention: H={H}, W={W}, {heads} heads of {C // max(heads, 1)} are not supported by the "
                         "native kernels (partition 7, head dim 32, H = W a multiple of 7)")
    _check_rows(qkv, N * H * W, 3 * C, "qkv")
    if table.dtype != torch.float32 or tuple(table.shape) != (169, heads) or not table.is_contiguous():
        raise ValueError(f"grid_attention: table must be the contiguous fp32 [169, {heads}] parameter")
    return C


def grid_attention_fwd(qkv: torch.Tensor, table: torch.Tensor, heads: int, N: int, H: int, W: int, scale: float,
                       grid: bool = True):
    """MaxViT's partition attention (7 x 7 sequences, head dim 32) on the image-order qkv rows [N*H*W, 3C] with the
    relative-position bias ``table`` [169, heads] fp32 and logits q . k * ``scale``: the grid partition (sequence (i, j)
    holds the pixels (a H/7 + i, b H/7 + j)), or with ``grid=False`` the window partition (pixels (7i + a, 7j + b)).
    Returns (O [N*H*W, C] in image order, lse fp32 [N*H*W, heads])."""
    C = _grid_check(qkv, table, heads, N, H, W)
    o = torch.empty((N * H * W, C), dtype=torch.bfloat16, device=qkv.device)
    lse = torch.empty((N * H * W, heads), dtype=torch.float32, device=qkv.device)
    _C().grid_attention_fwd(qkv.data_ptr(), table.data_ptr(), o.data_ptr(), lse.data_ptr(), N, H, W, heads, C,
                            bool(grid), float(scale), _stream())
    return o, lse


def grid_attention_bwd(dout: torch.Tensor, qkv: torch.Tensor, table: torch.Tensor, o: torch.Tensor, lse: torch.Tensor,
                       heads: int, N: int, H: int, W: int, scale: float, grad_table: Optional[torch.Tensor],
                       grid: bool = True) -> torch.Tensor:
    """dqkv [N*H*W, 3C] (qkv's layout) of :func:`grid_attention_fwd`; grad_table [169, heads] += the bias gradient
    (optional).  Deterministic: no atomics."""
    C = _grid_check(qkv, table, heads, N, H, W)
    _check_rows(o, N * H * W, C, "o")
    _check_rows(dout, N * H * W, C, "dout")
    if lse.dtype != torch.float32 or tuple(lse.shape) != (N * H * W, heads) or not lse.is_contiguous():
        raise ValueError("grid_attention_bwd: lse must be the contiguous fp32 [N*H*W, heads] of the forward")
    if grad_table is not None and (grad_table.dtype != torch.float32 or tuple(grad_table.shape) != (169, heads)
                                   or not grad_table.is_contiguous()):
        raise ValueError("grid_attention_bwd: grad_table must be a contiguous fp32 [169, heads] buffer")
    dqkv = torch.empty_like(qkv)
    scratch = torch.empty(_C().grid_attention_bwd_scratch_floats(N, H, heads), dtype=torch.float32, device=qkv.device)
    _C().grid_attention_bwd(qkv.data_ptr(), table.data_ptr(), o.data_ptr(), dout.data_ptr(), lse.data_ptr(),
                            dqkv.data_ptr(), _ptr(grad_table), scratch.data_ptr(), N, H, W, heads, C, bool(grid),
                            float(scale), _stream())
    return dqkv


def _merge_check(x: torch.Tensor) -> Tuple[int, int, int, int]:
    _check_act(x)
    _check_aligned(x, "x")
    N, C, H, W = x.shape
    if not supports_patch_merge(H, W, C):
        raise ValueError(f"patch_merge: an [N, {C}, {H}, {W}] map is not supported by the native kernels")
    return N, C, H, W


def patch_merge_fwd(x: torch.Tensor, gamma: torch.Tensor, beta: torch.Tensor, eps: float):
    """LayerNorm over 4C of the 2x2 gather (x[0::2, 0::2], x[1::2, 0::2], x[0::2, 1::2], x[1::2, 1::2]) of the NHWC
    activation x [N, C, H, W]: returns (rows bf16 [N*H/2*W/2, 4C], mean fp32 [rows], rstd fp32 [rows])."""
    N, C, H, W = _merge_check(x)
    _check_f32_vec(gamma, 4 * C, "gamma")
    _check_f32_vec(beta, 4 * C, "beta")
    M = N * (H // 2) * (W // 2)
    y = torch.empty((M, 4 * C), dtype=torch.bfloat16, device=x.device)
    mean = torch.empty(M, dtype=torch.float32, device=x.device)
    rstd = torch.empty(M, dtype=torch.float32, device=x.device)
    _C().patch_merge_fwd(x.data_ptr(), gamma.data_ptr(), beta.data_ptr(), y.data_ptr(), mean.data_ptr(), rstd.data_ptr(),
                         N, H, W, C, float(eps), sm_count(x.device.index or 0), _stream())
    return y, mean, rstd


def patch_merge_bwd(dy: torch.Tensor, x: torch.Tensor, mean: torch.Tensor, rstd: torch.Tensor, gamma: torch.Tensor,
                    grad_gamma: Optional[torch.Tensor], grad_beta: Optional[torch.Tensor]) -> torch.Tensor:
    """dx (like x) of :func:`patch_merge_fwd` from dy [rows, 4C]; grad_gamma / grad_beta [4C] += fixed-order sums."""
    N, C, H, W = _merge_check(x)
    M = N * (H // 2) * (W // 2)
    _check_rows(dy, M, 4 * C, "dy")
    _check_f32_vec(mean, M, "mean")
    _check_f32_vec(rstd, M, "rstd")
    for t, name in ((gamma, "gamma"), (grad_gamma, "grad_gamma"), (grad_beta, "grad_beta")):
        _check_f32_vec(t, 4 * C, name)
    sms = sm_count(x.device.index or 0)
    dx = torch.empty_like(x)
    scratch = torch.empty(_C().patch_merge_bwd_blocks(sms) * 8 * C, dtype=torch.float32, device=x.device)
    _C().patch_merge_bwd(dy.data_ptr(), x.data_ptr(), mean.data_ptr(), rstd.data_ptr(), gamma.data_ptr(), dx.data_ptr(),
                         _ptr(grad_gamma), _ptr(grad_beta), scratch.data_ptr(), N, H, W, C, sms, _stream())
    return dx


# ------------------------------------------------------------------------------------------------
# Swin V2: scaled-cosine window attention (csrc/ops/window_attention_v2.cu), continuous position bias and the
# patch-merging gather (csrc/ops/swin_v2.cu)
# ------------------------------------------------------------------------------------------------
def supports_window_attention_v2(H: int, W: int, window: int, heads: int, head_dim: int) -> bool:
    """Shapes the cosine window-attention kernels take: window 8, head dim 32, 1 to 32 heads (the CPB kernels' limit),
    any H and W (padded maps included)."""
    return window == 8 and head_dim == 32 and 0 < heads <= 32 and H > 0 and W > 0


def _win2_check(qkv, table, scale, qb, vb, heads, N, H, W, shift):
    C = qkv.shape[1] // 3 if qkv.dim() == 2 else 0
    if C == 0 or C % heads != 0 or not supports_window_attention_v2(H, W, 8, heads, C // heads):
        raise ValueError(f"window_attention_v2: H={H}, W={W}, {heads} heads of {C // max(heads, 1)} are not supported by "
                         "the native kernels (window 8, head dim 32, at most 32 heads)")
    if not 0 <= shift < 8:
        raise ValueError("window_attention_v2: shift must be in [0, 8)")
    _check_rows(qkv, N * H * W, 3 * C, "qkv")
    if table.dtype != torch.float32 or tuple(table.shape) != (225, heads) or not table.is_contiguous():
        raise ValueError(f"window_attention_v2: table must be a contiguous fp32 [225, {heads}] tensor")
    _check_f32_vec(scale, heads, "logit_scale")
    _check_f32_vec(qb, C, "q_bias")
    _check_f32_vec(vb, C, "v_bias")
    return C


def window_attention_v2_fwd(qkv: torch.Tensor, table: torch.Tensor, scale: torch.Tensor, qb: Optional[torch.Tensor],
                            vb: Optional[torch.Tensor], heads: int, N: int, H: int, W: int, shift: int):
    """Scaled-cosine shifted-window attention (window 8, head dim 32) on the image-order qkv rows [N*H*W, 3C] with the
    position-bias ``table`` [225, heads] and ``logit_scale`` [heads] fp32; padding tokens of a map whose sides are not
    multiples of 8 have q = ``qb``, k = 0, v = ``vb`` (fp32 [C] or None).  Returns (O [N*H*W, C] in image order, lse
    fp32 [N*H*W, heads])."""
    C = _win2_check(qkv, table, scale, qb, vb, heads, N, H, W, shift)
    sy, sx = window_shift(H, W, 8, shift)
    o = torch.empty((N * H * W, C), dtype=torch.bfloat16, device=qkv.device)
    lse = torch.empty((N * H * W, heads), dtype=torch.float32, device=qkv.device)
    _C().window_attention_v2_fwd(qkv.data_ptr(), table.data_ptr(), scale.data_ptr(), _ptr(qb), _ptr(vb), o.data_ptr(),
                                 lse.data_ptr(), N, H, W, heads, C, sy, sx, _stream())
    return o, lse


def window_attention_v2_bwd(dout: torch.Tensor, qkv: torch.Tensor, table: torch.Tensor, scale: torch.Tensor,
                            qb: Optional[torch.Tensor], vb: Optional[torch.Tensor], o: torch.Tensor, lse: torch.Tensor,
                            heads: int, N: int, H: int, W: int, shift: int, grad_table: Optional[torch.Tensor],
                            grad_scale: Optional[torch.Tensor], grad_bias: Optional[torch.Tensor],
                            bias_pad_only: bool = False) -> torch.Tensor:
    """dqkv [N*H*W, 3C] (qkv's layout) of :func:`window_attention_v2_fwd`.  Optional: grad_table [225, heads] = the
    table gradient (overwritten), grad_scale [heads] += the logit-scale gradient (0 where the clamp at ln 100 is active),
    grad_bias [3C] q and v slices += the bias gradients (the k slice is left as it is).  The bias sums cover every token,
    padding included: the gradient of b_q / b_v when qkv carries [b_q, 0, b_v] on every row.  ``bias_pad_only``: they
    cover the padding tokens only, the gradient of ``qb`` / ``vb`` as the padding fill of given qkv rows.
    Deterministic: no atomics."""
    C = _win2_check(qkv, table, scale, qb, vb, heads, N, H, W, shift)
    sy, sx = window_shift(H, W, 8, shift)
    _check_rows(o, N * H * W, C, "o")
    _check_rows(dout, N * H * W, C, "dout")
    if lse.dtype != torch.float32 or tuple(lse.shape) != (N * H * W, heads) or not lse.is_contiguous():
        raise ValueError("window_attention_v2_bwd: lse must be the contiguous fp32 [N*H*W, heads] of the forward")
    if grad_table is not None and (grad_table.dtype != torch.float32 or tuple(grad_table.shape) != (225, heads)
                                   or not grad_table.is_contiguous()):
        raise ValueError("window_attention_v2_bwd: grad_table must be a contiguous fp32 [225, heads] buffer")
    _check_f32_vec(grad_scale, heads, "grad_scale")
    _check_f32_vec(grad_bias, 3 * C, "grad_bias")
    dqkv = torch.empty_like(qkv)
    scratch = torch.empty(_C().window_attention_v2_bwd_scratch_floats(N, H, heads), dtype=torch.float32,
                          device=qkv.device)
    _C().window_attention_v2_bwd(qkv.data_ptr(), table.data_ptr(), scale.data_ptr(), _ptr(qb), _ptr(vb), o.data_ptr(),
                                 dout.data_ptr(), lse.data_ptr(), dqkv.data_ptr(), _ptr(grad_table), _ptr(grad_scale),
                                 _ptr(grad_bias), scratch.data_ptr(), N, H, W, heads, C, sy, sx, bool(bias_pad_only),
                                 _stream())
    return dqkv


def _cpb_check(coords, w1, b1, w2, heads):
    if not 0 < heads <= 32:
        raise ValueError("cpb: 1 to 32 heads")
    _check_f32_vec(coords, 450, "relative_coords_table")
    _check_f32_vec(w1, 1024, "cpb_mlp.0.weight")
    _check_f32_vec(b1, 512, "cpb_mlp.0.bias")
    _check_f32_vec(w2, 512 * heads, "cpb_mlp.2.weight")


def cpb_fwd(coords: torch.Tensor, w1: torch.Tensor, b1: torch.Tensor, w2: torch.Tensor, heads: int,
            qkv_b: Optional[torch.Tensor] = None):
    """The continuous position-bias table [225, heads] fp32 = 16 sigmoid(cpb_mlp(relative_coords_table)); with
    ``qkv_b`` [3C], also returns it with the k slice zeroed (the bias the qkv linear runs with), else None."""
    _cpb_check(coords, w1, b1, w2, heads)
    table = torch.empty((225, heads), dtype=torch.float32, device=coords.device)
    eff = None
    if qkv_b is not None:
        _check_f32_vec(qkv_b, qkv_b.numel(), "qkv_b")
        eff = torch.empty_like(qkv_b)
    _C().cpb_fwd(coords.data_ptr(), w1.data_ptr(), b1.data_ptr(), w2.data_ptr(), table.data_ptr(), _ptr(qkv_b),
                 _ptr(eff), heads, 0 if qkv_b is None else qkv_b.numel() // 3, _stream())
    return table, eff


def cpb_bwd(coords: torch.Tensor, w1: torch.Tensor, b1: torch.Tensor, w2: torch.Tensor, table: torch.Tensor,
            grad_table: torch.Tensor, heads: int, grad_w1: Optional[torch.Tensor], grad_b1: Optional[torch.Tensor],
            grad_w2: Optional[torch.Tensor]) -> None:
    """grad_w1 [512, 2], grad_b1 [512], grad_w2 [heads, 512] += the CPB MLP's gradients from grad_table [225, heads] and
    the forward's ``table`` (each optional; fixed order, two kernels)."""
    _cpb_check(coords, w1, b1, w2, heads)
    _check_f32_vec(table, 225 * heads, "table")
    _check_f32_vec(grad_table, 225 * heads, "grad_table")
    for t, n, name in ((grad_w1, 1024, "grad_w1"), (grad_b1, 512, "grad_b1"), (grad_w2, 512 * heads, "grad_w2")):
        _check_f32_vec(t, n, name)
    scratch = torch.empty(_C().cpb_bwd_scratch_floats(heads), dtype=torch.float32, device=coords.device)
    _C().cpb_bwd(coords.data_ptr(), w1.data_ptr(), b1.data_ptr(), w2.data_ptr(), table.data_ptr(), grad_table.data_ptr(),
                 _ptr(grad_w1), _ptr(grad_b1), _ptr(grad_w2), scratch.data_ptr(), heads, _stream())


def merge_gather(x: torch.Tensor) -> torch.Tensor:
    """The 2x2 gather (x[0::2, 0::2], x[1::2, 0::2], x[0::2, 1::2], x[1::2, 1::2]) of the NHWC activation x [N, C, H, W]
    (H, W even, C % 8 == 0) as rows bf16 [N*H/2*W/2, 4C]."""
    _check_act(x)
    _check_aligned(x, "x")
    N, C, H, W = x.shape
    if H % 2 or W % 2 or C % 8:
        raise ValueError(f"merge_gather: an [N, {C}, {H}, {W}] map is not supported (H, W even, C % 8 == 0)")
    y = torch.empty((N * (H // 2) * (W // 2), 4 * C), dtype=torch.bfloat16, device=x.device)
    _C().merge_gather(x.data_ptr(), y.data_ptr(), N, H, W, C, True, sm_count(x.device.index or 0), _stream())
    return y


def merge_scatter(dy: torch.Tensor, N: int, C: int, H: int, W: int) -> torch.Tensor:
    """Backward of :func:`merge_gather`: dx [N, C, H, W] (channels_last) from dy [N*H/2*W/2, 4C]."""
    if H % 2 or W % 2 or C % 8:
        raise ValueError(f"merge_scatter: an [N, {C}, {H}, {W}] map is not supported (H, W even, C % 8 == 0)")
    _check_rows(dy, N * (H // 2) * (W // 2), 4 * C, "dy")
    dx = torch.empty((N, C, H, W), dtype=torch.bfloat16, device=dy.device, memory_format=torch.channels_last)
    _C().merge_gather(dy.data_ptr(), dx.data_ptr(), N, H, W, C, False, sm_count(dy.device.index or 0), _stream())
    return dx


# ------------------------------------------------------------------------------------------------
# squeeze-excitation (csrc/ops/squeeze_excite.cu) and hardswish on [B, F]
# ------------------------------------------------------------------------------------------------
def _check_gate(s: torch.Tensor, n: int, c: int) -> None:
    """``s``: the fc2 output [N, >= C] bf16 (row stride a multiple of 8, unit column stride)."""
    if s.dtype != torch.bfloat16 or not s.is_cuda or s.dim() != 2 or s.shape[0] != n or s.shape[1] < c \
            or s.stride(1) != 1 or s.stride(0) % 8 != 0 or s.stride(0) < c:
        raise ValueError(f"squeeze-excite: expected the CUDA bf16 gate logits [N={n}, >= {c}] with a row stride that is a "
                         "multiple of 8")
    _check_aligned(s, "s")


def _check_se_act(x: torch.Tensor, name: str) -> None:
    _check_act(x, name)
    if x.dim() != 4 or x.shape[1] % 8 != 0:
        raise ValueError(f"{name}: squeeze-excite needs a 4-D activation with a multiple of 8 channels")
    _check_aligned(x, name)


_SE_GATES = ("hardsigmoid", "sigmoid")


def _se_kernel(name: str, gate: str):
    """The hardsigmoid kernels (squeeze_excite.cu) or the sigmoid ones (squeeze_excite_sigmoid.cu)."""
    if gate not in _SE_GATES:
        raise ValueError(f"squeeze-excite: gate must be one of {_SE_GATES}, got {gate!r}")
    return getattr(_C(), name if gate == "hardsigmoid" else name.replace("se_", "se_sig_"))


def se_scale(x: torch.Tensor, s: torch.Tensor, gate: str = "hardsigmoid") -> torch.Tensor:
    """y = x * gate(s[n, c]) for an NHWC activation x [N, C, H, W] and the gate logits s [N, >= C]; ``gate`` is
    "hardsigmoid" (MobileNetV3) or "sigmoid" (EfficientNet)."""
    _check_se_act(x, "x")
    N, Ch, H, W = x.shape
    _check_gate(s, N, Ch)
    y = torch.empty_like(x)
    _se_kernel("se_scale", gate)(x.data_ptr(), s.data_ptr(), s.stride(0), y.data_ptr(), N, H * W, Ch, sm_count(x.device.index or 0),
                  _stream())
    return y


def se_reduce(dy: torch.Tensor, x: torch.Tensor, s: torch.Tensor, gate: str = "hardsigmoid") -> torch.Tensor:
    """ds [N, C rounded up to 64] bf16 = gate'(s) * sum_hw(dy * x), pad columns zero: the gradient of the gate
    logits of :func:`se_scale`, laid out as the fc2 GEMM operand.  Deterministic (no atomics).  The sigmoid's
    derivative is g (1 - g), g = sigmoid(s) recomputed from the saved logits."""
    _check_se_act(dy, "dy")
    _check_se_act(x, "x")
    N, Ch, H, W = x.shape
    if tuple(dy.shape) != tuple(x.shape):
        raise ValueError("se_reduce: dy and x differ in shape")
    _check_gate(s, N, Ch)
    ldd = _ceil_div(Ch, 64) * 64
    ds = torch.empty((N, ldd), dtype=torch.bfloat16, device=x.device)
    _se_kernel("se_reduce", gate)(dy.data_ptr(), x.data_ptr(), s.data_ptr(), s.stride(0), ds.data_ptr(), ldd, N, H * W,
                                   Ch, _stream())
    return ds


def se_apply(dy: torch.Tensor, s: torch.Tensor, dpooled: torch.Tensor, gate: str = "hardsigmoid") -> torch.Tensor:
    """dx = dy * gate(s[n, c]) + dpooled[n, c] / (H*W): the input gradient of squeeze-excitation from both of its
    paths (the scale and the pooling) in one pass."""
    _check_se_act(dy, "dy")
    N, Ch, H, W = dy.shape
    _check_gate(s, N, Ch)
    if dpooled.dtype != torch.bfloat16 or tuple(dpooled.shape) != (N, Ch) or not dpooled.is_contiguous():
        raise ValueError(f"se_apply: expected a contiguous bf16 dpooled [{N}, {Ch}]")
    _check_aligned(dpooled, "dpooled")
    dx = torch.empty_like(dy)
    _se_kernel("se_apply", gate)(dy.data_ptr(), s.data_ptr(), s.stride(0), dpooled.data_ptr(), dx.data_ptr(), N, H * W,
                                  Ch, sm_count(dy.device.index or 0), _stream())
    return dx


def pad_cols_bf16(w: torch.Tensor, kp: int) -> torch.Tensor:
    """bf16 [rows, k] -> [rows, kp] with zero columns [k, kp): fc2's weight with its squeeze dimension padded to a
    multiple of 8, so that its rows are 16-byte GEMM operand rows."""
    if w.dtype != torch.bfloat16 or w.dim() != 2 or kp < w.shape[1]:
        raise ValueError(f"pad_cols_bf16: expected a contiguous CUDA bf16 matrix with at most {kp} columns")
    return pad_cols([(w, w.shape[0], kp)])[0]


def pad_cols(mats) -> list:
    """Zero-padded copies of up to 24 matrices in ONE launch: ``mats`` = [(src, prows, kp)] with ``src`` a contiguous
    CUDA bf16 or fp32 tensor viewed as [rows, k] (its first dimension, the rest flattened; a vector is one row), and the
    result for each a new [prows, kp] tensor of the same dtype holding ``src`` in its top-left corner, zeros elsewhere.
    An entry (src, prows, kp, dst) writes into ``dst`` instead (a contiguous [prows, kp] tensor, for instance a row
    slice of a stacked matrix), which is also the result."""
    out, desc = [], []
    for entry in mats:
        src, prows, kp = entry[:3]
        dst = entry[3] if len(entry) > 3 else None
        rows, k = (1, src.numel()) if src.dim() == 1 else (src.shape[0], src.numel() // max(1, src.shape[0]))
        if src.dtype not in (torch.bfloat16, torch.float32) or not src.is_cuda or not src.is_contiguous() \
                or prows < rows or kp < k or rows <= 0 or k <= 0:
            raise ValueError(f"pad_cols: expected contiguous CUDA bf16 / fp32 matrices of at most [{prows}, {kp}], got "
                             f"{tuple(src.shape)} {src.dtype}")
        if dst is None:
            dst = torch.empty((prows, kp), dtype=src.dtype, device=src.device)
        elif dst.dtype != src.dtype or not dst.is_contiguous() or dst.numel() != prows * kp or dst.device != src.device:
            raise ValueError(f"pad_cols: the destination must be a contiguous {src.dtype} tensor of {prows} x {kp}")
        out.append(dst)
        desc.append((src.data_ptr(), dst.data_ptr(), rows, k, prows, kp, src.element_size()))
    if not 0 < len(desc) <= 24:
        raise ValueError("pad_cols: 1 to 24 matrices per launch")
    _C().pad_cols(desc, _stream())
    return out


def fold_cols_f32(src: torch.Tensor, dst: torch.Tensor) -> None:
    """dst [rows, k] (fp32, any contiguous shape of rows * k elements) += src [rows, kp][:, :k]."""
    fold_cols([(src, dst, src.shape[0])])


def fold_cols(mats, add: bool = True) -> None:
    """ONE launch over up to 24 pairs ``(src [prows, kp], dst, rows)``: fp32 ``dst`` (contiguous, rows * k elements)
    += ``src[:rows, :k]`` (``add``), or = it (the running statistics of a padded BatchNorm)."""
    desc = []
    for src, dst, rows in mats:
        if src.dim() == 1:
            src = src.view(1, -1)
        if src.dtype != torch.float32 or dst.dtype != torch.float32 or not src.is_contiguous() \
                or not dst.is_contiguous() or rows <= 0 or rows > src.shape[0] or dst.numel() % rows != 0 \
                or dst.numel() // rows > src.shape[1]:
            raise ValueError("fold_cols: expected contiguous fp32 src [prows, kp] and dst [rows <= prows, k <= kp]")
        desc.append((src.data_ptr(), dst.data_ptr(), rows, dst.numel() // rows, src.shape[1], int(add)))
    if not 0 < len(desc) <= 24:
        raise ValueError("fold_cols: 1 to 24 matrices per launch")
    _C().fold_cols(desc, _stream())


def silu_rows_fwd(x: torch.Tensor, cols: int) -> torch.Tensor:
    """y [N, cols] = silu(x[:, :cols]) for a bf16 matrix x [N, ld] (cols <= ld, both multiples of 8)."""
    _check_act(x, "x")
    if x.dim() != 2 or x.shape[1] % 8 != 0 or cols % 8 != 0 or not 0 < cols <= x.shape[1]:
        raise ValueError("silu_rows_fwd: expected a bf16 [N, ld] matrix and cols <= ld, both multiples of 8")
    y = torch.empty((x.shape[0], cols), dtype=torch.bfloat16, device=x.device)
    _C().silu_rows_fwd(x.data_ptr(), x.shape[1], y.data_ptr(), cols, x.shape[0], _stream())
    return y


def silu_rows_bwd(dy: torch.Tensor, x: torch.Tensor, c_valid: int) -> torch.Tensor:
    """dx [N, ld] = dy * silu'(x) in columns < c_valid and 0 beyond, for the saved pre-activation x [N, ld] and
    dy [N, <= ld]: the gradient of :func:`silu_rows_fwd` laid out as a zero-padded GEMM operand."""
    _check_act(dy, "dy")
    _check_act(x, "x")
    if dy.dim() != 2 or x.dim() != 2 or dy.shape[0] != x.shape[0] or dy.shape[1] % 8 != 0 or x.shape[1] % 8 != 0 \
            or dy.shape[1] > x.shape[1] or not 0 < c_valid <= dy.shape[1]:
        raise ValueError("silu_rows_bwd: expected bf16 dy [N, k] and x [N, ld >= k] (multiples of 8), 0 < c_valid <= k")
    dx = torch.empty_like(x)
    _C().silu_rows_bwd(dy.data_ptr(), dy.shape[1], x.data_ptr(), x.shape[1], dx.data_ptr(), c_valid, x.shape[0], _stream())
    return dx


def stochastic_depth_keep(n: int, p: float, seed: int, offset: int, step: Optional[torch.Tensor], device) -> torch.Tensor:
    """fp32 [n] per-sample scales, 0 or 1 / (1 - p), drawn on the device from the dropout Philox stream (``step``: the
    device step counter mixed into the key, see :func:`dropout`)."""
    if not 0.0 < p < 1.0 or n <= 0:
        raise ValueError(f"stochastic_depth_keep: need n > 0 and 0 < p < 1, got n={n}, p={p}")
    keep = torch.empty(n, dtype=torch.float32, device=device)
    _C().stochastic_depth_keep(keep.data_ptr(), n, p, seed, offset, _stream(), _ptr(step))
    return keep


def _check_flat(t: torch.Tensor, name: str) -> None:
    if t.dtype != torch.bfloat16 or not t.is_cuda or not t.is_contiguous() or t.numel() % 8 != 0:
        raise ValueError(f"{name}: expected a contiguous CUDA bf16 tensor with a multiple of 8 elements")
    _check_aligned(t, name)


def hardswish_fwd(x: torch.Tensor) -> torch.Tensor:
    """y = x * clamp(x + 3, 0, 6) / 6 elementwise (MobileNetV3's classifier activation)."""
    _check_flat(x, "x")
    y = torch.empty_like(x)
    _C().hardswish_fwd(x.data_ptr(), y.data_ptr(), x.numel(), _stream())
    return y


def hardswish_bwd(dy: torch.Tensor, x: torch.Tensor) -> torch.Tensor:
    """dx = dy * hardswish'(x), x being the saved pre-activation."""
    _check_flat(dy, "dy")
    _check_flat(x, "x")
    if dy.shape != x.shape:
        raise ValueError("hardswish_bwd: dy and x differ in shape")
    dx = torch.empty_like(dy)
    _C().hardswish_bwd(dy.data_ptr(), x.data_ptr(), dx.data_ptr(), x.numel(), _stream())
    return dx


def tanh_rows_fwd(x: torch.Tensor) -> torch.Tensor:
    """y = tanh(x) elementwise (MaxViT's classifier activation)."""
    _check_flat(x, "x")
    y = torch.empty_like(x)
    _C().tanh_rows_fwd(x.data_ptr(), y.data_ptr(), x.numel(), _stream())
    return y


def tanh_rows_bwd(dy: torch.Tensor, y: torch.Tensor) -> torch.Tensor:
    """dx = dy * (1 - y^2), y being the saved output of :func:`tanh_rows_fwd`."""
    _check_flat(dy, "dy")
    _check_flat(y, "y")
    if dy.shape != y.shape:
        raise ValueError("tanh_rows_bwd: dy and y differ in shape")
    dx = torch.empty_like(dy)
    _C().tanh_rows_bwd(dy.data_ptr(), y.data_ptr(), dx.data_ptr(), y.numel(), _stream())
    return dx


def expand_grouped_weight(w_bf16: torch.Tensor, taps: int, groups: int) -> torch.Tensor:
    """Compact grouped weights ``[Cout, taps * cg]`` bf16 (KRSC of ``[Cout, cg, R, S]``) -> the operand of the grouped
    kernels, laid out per group bundle (:func:`grouped_bundle`: Wb channels, T tiles):
    ``[nbundles * T * 64, taps * T * 64]``.  Row ``b * T * 64 + l`` (``l < Wb``) belongs to output channel
    ``co = b * Wb + l`` and holds its ``cg`` input channels of each tap at columns ``tap * T * 64 + (l - l % cg) + j``;
    everything else is zero, including the rows ``l >= Wb`` that the data gradient's K overhang reads.  At Wb = 64 this
    is ``[Cout, taps * 64]`` with columns ``tap * 64 + (co % 64 - co % cg) + j``.  Made once per step, in forward (so
    that a captured graph re-derives it from the weights every replay), and kept for that step's data gradient."""
    cout = w_bf16.shape[0]
    cg = cout // groups
    if w_bf16.dtype != torch.bfloat16 or w_bf16.numel() != cout * taps * cg or not w_bf16.is_contiguous():
        raise ValueError("expand_grouped_weight: expected contiguous bf16 [Cout, taps * Cout / groups] weights")
    out = torch.empty(grouped_expanded_shape(cout, taps, groups), dtype=torch.bfloat16, device=w_bf16.device)
    _C().expand_grouped_weight(w_bf16.data_ptr(), out.data_ptr(), cout, taps, cg, _stream())
    return out


def expand_grouped_weight_ref(w: torch.Tensor, taps: int, groups: int) -> torch.Tensor:
    """Torch twin of :func:`expand_grouped_weight` (any device and dtype), index by index from the bundle layout: the
    reference the kernel is checked against."""
    cout = w.shape[0]
    cg = cout // groups
    wb, t = grouped_bundle(cg)
    out = w.new_zeros(grouped_expanded_shape(cout, taps, groups))
    wc = w.reshape(cout, taps, cg)
    co = torch.arange(cout, device=w.device)
    l = co % wb                                       # position in the bundle
    row = co // wb * t * 64 + l
    col0 = l - l % cg                                 # first column of co's group inside a tap's 64 T
    for tap in range(taps):
        for j in range(cg):
            out[row, tap * t * 64 + col0 + j] = wc[:, tap, j]
    return out


def _check_grouped(cin: int, cout: int, groups: int, w_bf16: torch.Tensor, taps: int) -> None:
    if not grouped_conv_native(cin, cout, groups):
        raise ValueError(f"grouped conv {cin} -> {cout} in {groups} groups is not supported by the native kernels")
    if tuple(w_bf16.shape) != grouped_expanded_shape(cout, taps, groups):
        raise ValueError("grouped conv: pass the expanded weights of expand_grouped_weight")


def _conv_grouped(mode: int, src: torch.Tensor, out: torch.Tensor, w_bf16: torch.Tensor, C: int, M: int, srcHW, dstHW,
                  kernel, stride: int, ph: int, pw: int, dil: int, groups: int, s_ptr: int = 0, ss_ptr: int = 0,
                  batch: int = 0, tile=(0, 0, 0), zfill: int = 0, variant: int = 0) -> None:
    """One launch of the grouped kernels (forward: tile / gather fwd; data gradient: tile / gather dgrad) with T
    64-channel k-blocks per tap (:func:`grouped_bundle`)."""
    R, S = kernel
    wb, t = grouped_bundle(C // groups)
    rows, cols = w_bf16.shape
    tma = mode in (_C().CONV_TILE_FWD, _C().CONV_TILE_DGRAD)
    _C().conv_gemm(mode, 0 if tma else src.data_ptr(), out.data_ptr(), 0, 0, s_ptr, ss_ptr, M, R * S * t, C, srcHW[0],
                   srcHW[1], C, dstHW[0], dstHW[1], R, S, stride, ph, dil, t, 0, C, w_bf16.data_ptr(), rows, cols, rows,
                   src.data_ptr() if tma else 0, C if tma else 0, batch, tile[0], tile[1], tile[2], zfill, _stream(), pw,
                   t * 64, variant=variant, grouped=wb)


# ------------------------------------------------------------------------------------------------
# convolution forward / dgrad / wgrad
# ------------------------------------------------------------------------------------------------
def conv_fwd(x: torch.Tensor, w_bf16: torch.Tensor, kernel: Tuple[int, int], stride: int, pad, dil: int = 1,
             stats: bool = False, bias: Optional[torch.Tensor] = None, relu: bool = False,
             cout: Optional[int] = None, prepadded: Optional[torch.Tensor] = None, groups: int = 1):
    """y = conv(x, w) [+ bias][ReLU]; optionally per-channel (sum, sumsq) of y for BatchNorm.
    ``prepadded``: result of :func:`stem_prepare` for this (x, geometry) — skips the internal padding copy.

    ``w_bf16``: [Cout, R*S*Cin] bf16 (or the packed stem matrix [Cout, KB*64]); ``pad``: int or (pad_h, pad_w).
    ``groups`` > 1: a grouped convolution (:func:`grouped_conv_native`); ``w_bf16`` is then the expanded matrix of
    :func:`expand_grouped_weight`; no bias / ReLU.
    """
    C = _C()
    _check_act(x)
    N, Cin, H, W = x.shape
    R, S = kernel
    ph, pw = _pad2(pad)
    Cout = cout if cout is not None else (Cin if groups > 1 else w_bf16.shape[0])   # grouped: Cin = Cout
    if Cout % 8 != 0:
        raise ValueError("conv_fwd: Cout must be a multiple of 8")
    P, Q = conv_out_hw(H, W, kernel, stride, (ph, pw), dil)
    M = N * P * Q
    y = empty_act(N, Cout, P, Q, x.device)
    st = zeros_f32((2, Cout), x.device) if stats else None
    s_ptr, ss_ptr = (st[0].data_ptr(), st[1].data_ptr()) if stats else (0, 0)
    if groups > 1:
        _check_grouped(Cin, Cout, groups, w_bf16, R * S)
        if bias is not None or relu:
            raise ValueError("conv_fwd: grouped convolutions take no bias / ReLU epilogue")
        geo = dict(srcHW=(H, W), dstHW=(P, Q), kernel=kernel, stride=stride, ph=ph, pw=pw, dil=dil, groups=groups,
                   s_ptr=s_ptr, ss_ptr=ss_ptr, batch=N)
        if USE_TILE_TMA and (stride == 1 or (stride == 2 and R * S <= 16 and USE_TILE_S2)):
            tile = tile_geometry(P, Q, N, 128)
            t = grouped_bundle(Cin // groups)[1]
            _tuned(("fwd_g", N, H, W, Cin, Cout, R, S, stride, ph, pw, dil, stats, groups),
                   conv_variants(w_bf16.shape[0], M, R * S * t, False, grouped=True),
                   lambda v: _conv_grouped(C.CONV_TILE_FWD, x, y, w_bf16, Cout, M, tile=tile, variant=v, **geo),
                   (st,) if stats else ())
        else:
            _conv_grouped(C.CONV_FWD, x, y, w_bf16, Cout, M, **geo)
        return (y, st) if stats else y
    n_total = _ceil_div(Cout, 64) * 64              # N tiles cover the padded width; stores / stats stop at Cout
    cch = _ceil_div(Cin, 64)
    wp, wr, wc = w_bf16.data_ptr(), w_bf16.shape[0], w_bf16.shape[1]
    if Cin <= 4:
        if Cin != 4:
            raise ValueError("stem input must be padded to 4 channels (NHWC4)")
        SP, RPK, KB, RP = stem_geometry(R, S)
        geo = stem_tma_geometry(H, W, kernel, stride, (ph, pw)) if dil == 1 else None
        if geo is not None:
            # even stride: copy the image into a zero-bordered buffer once (one 8-byte-per-pixel pass) and let ONE
            # 5-D TMA box per k-block fetch what the gather path needs 64 cp.async per output pixel for
            xp = prepadded if prepadded is not None else pad_image(x, geo[0], geo[1], ph, pw, geo[2])
            tw, th, tn = tile_geometry(P, Q, N, 128)
            C.conv_gemm(C.CONV_STEM_TMA, 0, y.data_ptr(), 0, _ptr(bias), s_ptr, ss_ptr, M, KB, Cout, geo[0], geo[1], 4,
                        P, Q, R, S, stride, 0, 1, RPK, int(relu), Cout, wp, wr, wc, n_total, xp.data_ptr(), 4, N, tw, th,
                        tn, 0, _stream(), 0, 0)
        else:
            C.conv_gemm(C.CONV_STEM, x.data_ptr(), y.data_ptr(), 0, _ptr(bias), s_ptr, ss_ptr, M, KB, Cout, H, W, 4,
                        P, Q, R, S, stride, ph, dil, SP, int(relu), Cout, wp, wr, wc, n_total, 0, 0, N, 0, 0, 0, 0,
                        _stream(), pw, 0)
        return (y, st) if stats else y
    if Cin % 8 != 0:
        raise ValueError("conv_fwd: Cin must be a multiple of 8 (or an NHWC4 stem)")
    from . import fp8 as _fp8

    one_by_one = R == 1 and S == 1 and stride == 1 and ph == 0 and pw == 0
    tile_ok = USE_TILE_TMA and (stride == 1 or (stride == 2 and R * S <= 16 and USE_TILE_S2))
    if _fp8.fwd_eligible(Cin, Cout, R * S) and (one_by_one or tile_ok) and M >= 2048:
        # e4m3 operands: quantise x (delayed per-tensor scale) and take this step's e4m3 weights; a k-block is 128
        # channels (128 bytes), the epilogue multiplies by inv_scale(x) * inv_scale(w)
        tw_ = _fp8.twin_of(x)                       # produced by the BN-apply kernel that wrote x, if any
        if tw_ is None:
            _fp8.request_twin(x)                    # from the next step on the producer emits the e4m3 copy itself
        xq, sx = tw_ if tw_ is not None else _fp8.quantize(x, ("x", wp, N, H, W))
        wq, sw = _fp8.quantize_weight(w_bf16)
        cch8 = Cin // 128
        fp8kw = dict(fp8=1, deq_a=_fp8.inv_scale_ptr(sx, x.device), deq_b=_fp8.inv_scale_ptr(sw, x.device))
        cands = conv_variants(n_total, M, R * S * cch8, False, fp8=True)
        _fp8.count("fwd")
        if one_by_one:
            _tuned(("fwd1x1_f8", N, H, W, Cin, Cout, stats, bias is not None, relu), cands,
                   lambda v: C.conv_gemm(C.CONV_GEMM, 0, y.data_ptr(), 0, _ptr(bias), s_ptr, ss_ptr, M, cch8, Cout, H, W,
                                         Cin, P, Q, 1, 1, 1, 0, 1, cch8, int(relu), Cout, wq.data_ptr(), wr, wc, n_total,
                                         xq.data_ptr(), Cin, N, 0, 0, 0, 0, _stream(), 0, Cin, variant=v, **fp8kw),
                   (st,) if stats else ())
        else:
            tw, th, tn = tile_geometry(P, Q, N, 128)
            _tuned(("fwd_f8", N, H, W, Cin, Cout, R, S, stride, ph, pw, dil, stats, bias is not None, relu), cands,
                   lambda v: C.conv_gemm(C.CONV_TILE_FWD, 0, y.data_ptr(), 0, _ptr(bias), s_ptr, ss_ptr, M, R * S * cch8,
                                         Cout, H, W, Cin, P, Q, R, S, stride, ph, dil, cch8, int(relu), Cout,
                                         wq.data_ptr(), wr, wc, n_total, xq.data_ptr(), Cin, N, tw, th, tn, 0, _stream(),
                                         pw, Cin, variant=v, **fp8kw),
                   (st,) if stats else ())
        return (y, st) if stats else y
    if R == 1 and S == 1 and stride == 1 and ph == 0 and pw == 0:
        _tuned(("fwd1x1", N, H, W, Cin, Cout, stats, bias is not None, relu), conv_variants(n_total, M, cch, False),
               lambda v: C.conv_gemm(C.CONV_GEMM, 0, y.data_ptr(), 0, _ptr(bias), s_ptr, ss_ptr, M, cch, Cout, H, W, Cin,
                                     P, Q, 1, 1, 1, 0, 1, cch, int(relu), Cout, wp, wr, wc, n_total, x.data_ptr(), Cin,
                                     N, 0, 0, 0, 0, _stream(), 0, Cin, variant=v),
               (st,) if stats else ())
    elif USE_TILE_TMA and (stride == 1 or (stride == 2 and R * S <= 16 and USE_TILE_S2)):
        # window conv: the activation operand comes through ONE 4-D TMA box per filter tap (stride 2: the box is
        # taken from the matching 2x2 phase sub-image of x)
        tw, th, tn = tile_geometry(P, Q, N, 128)
        _tuned(("fwd", N, H, W, Cin, Cout, R, S, stride, ph, pw, dil, stats, bias is not None, relu),
               conv_variants(n_total, M, R * S * cch, False),
               lambda v: C.conv_gemm(C.CONV_TILE_FWD, 0, y.data_ptr(), 0, _ptr(bias), s_ptr, ss_ptr, M, R * S * cch,
                                     Cout, H, W, Cin, P, Q, R, S, stride, ph, dil, cch, int(relu), Cout, wp, wr, wc,
                                     n_total, x.data_ptr(), Cin, N, tw, th, tn, 0, _stream(), pw, Cin, variant=v),
               (st,) if stats else ())
    else:
        C.conv_gemm(C.CONV_FWD, x.data_ptr(), y.data_ptr(), 0, _ptr(bias), s_ptr, ss_ptr, M, R * S * cch,
                    Cout, H, W, Cin, P, Q, R, S, stride, ph, dil, cch, int(relu), Cout, wp, wr, wc, n_total, 0, 0,
                    N, 0, 0, 0, 0, _stream(), pw, Cin)
    return (y, st) if stats else y


def conv_dgrad(dy: torch.Tensor, w_bf16: torch.Tensor, x_shape, kernel: Tuple[int, int], stride: int, pad,
               dil: int = 1, add: Optional[torch.Tensor] = None, add_mask: Optional[torch.Tensor] = None,
               bn_reduce: Optional[tuple] = None, groups: int = 1) -> torch.Tensor:
    """dx = conv_transpose(dy, w) (+ add [gated by the bit mask ``add_mask``: uint8 [M, Cin/8]]).
    ``w_bf16`` is the forward matrix [Cout, R*S*Cin] (``groups`` > 1: the forward's :func:`expand_grouped_weight`).

    ``bn_reduce = (y, gamma, beta, save, scratch[, zmask])``: dx is the output gradient of a BN+ReLU layer whose saved
    input is ``y``; the kernel's epilogue then also accumulates that BN's dbeta / dgamma sums into ``scratch`` (fp32
    [2, Cin], zeroed), so ``bn_act_bwd(..., pre_reduced=scratch)`` can skip its reduction pass over (dx, y).  The ReLU
    mask is recomputed from ``y``, or, with ``zmask`` (the layer's forward bit mask, for a residual layer), read from it.
    With ``add`` (1x1 stride-1 only) the sums are over the stored value, the product plus the gated ``add``."""
    C = _C()
    _check_act(dy, "dy")
    N, Cin, H, W = x_shape
    _, Cout, P, Q = dy.shape
    R, S = kernel
    ph, pw = _pad2(pad)
    if Cin % 8 != 0 or Cout % 8 != 0:
        raise ValueError("conv_dgrad needs Cin, Cout multiples of 8")
    s2_tile = USE_TILE_TMA and USE_TILE_S2 and stride == 2 and R * S <= 16 and dil == 1 and add is None
    dx = empty_act(N, Cin, H, W, dy.device)
    zfill = 0
    if s2_tile:
        # output phases that receive no tap (e.g. 1x1 stride 2 only feeds even rows/cols; 3x3 stride 2 without
        # padding leaves none empty) and border rows/cols no window reaches.  Even image + 1x1: the live phase's
        # epilogue writes the zeros of its three sibling pixels; otherwise clear dx first.
        covered_h = (P - 1) * 2 + (R - 1) * dil + 1 - ph >= H
        covered_w = (Q - 1) * 2 + (S - 1) * dil + 1 - pw >= W
        if R == 1 and S == 1 and ph == 0 and pw == 0 and H % 2 == 0 and W % 2 == 0:
            zfill = 1
        elif R < 2 or S < 2 or not (covered_h and covered_w):
            dx.zero_()
    if groups > 1:
        # group bundles: an N tile of input channels of a bundle reads that bundle's dy channels and the expanded
        # weights MN-major; the shortcut add and the BN-backward reduction are not fused here
        _check_grouped(Cin, Cout, groups, w_bf16, R * S)
        if add is not None or add_mask is not None or bn_reduce is not None:
            raise ValueError("conv_dgrad: grouped convolutions take no add / add_mask / bn_reduce")
        geo = dict(srcHW=(P, Q), dstHW=(H, W), kernel=kernel, stride=stride, ph=ph, pw=pw, dil=dil, groups=groups,
                   batch=N)
        nt, t = w_bf16.shape[0], grouped_bundle(Cin // groups)[1]
        if stride == 1 and USE_TILE_TMA:
            tile = tile_geometry(H, W, N, 128)
            _tuned(("dgrad_g", N, H, W, Cin, Cout, R, S, 1, ph, pw, dil, groups),
                   conv_variants(nt, N * H * W, R * S * t, True, grouped=True),
                   lambda v: _conv_grouped(C.CONV_TILE_DGRAD, dy, dx, w_bf16, Cin, N * H * W, tile=tile, variant=v,
                                           **geo))
        elif s2_tile:
            tile = tile_geometry((H + 1) // 2, (W + 1) // 2, N, 128)
            _tuned(("dgrad_s2_g", N, H, W, Cin, Cout, R, S, 2, ph, pw, dil, zfill, groups),
                   conv_variants(nt, N * ((H + 1) // 2) * ((W + 1) // 2), max(1, (R * S * t) // 4), True, grouped=True),
                   lambda v: _conv_grouped(C.CONV_TILE_DGRAD, dy, dx, w_bf16, Cin, N * H * W, tile=tile, zfill=zfill,
                                           variant=v, **geo))
        else:
            _conv_grouped(C.CONV_DGRAD, dy, dx, w_bf16, Cin, N * H * W, **geo)
        return dx
    if add is not None:
        _check_act(add, "add")
    if add_mask is not None and (add is None or add_mask.dtype != torch.uint8 or add_mask.numel() != N * H * W * (Cin // 8)):
        raise ValueError("add_mask: expected a uint8 [N*H*W, Cin/8] bit mask accompanying `add`")
    n_total = _ceil_div(Cin, 64) * 64
    cch = _ceil_div(Cout, 64)
    wp, wr, wc = w_bf16.data_ptr(), w_bf16.shape[0], w_bf16.shape[1]
    bnr = {}
    s1 = s2 = 0
    one_by_one = R == 1 and S == 1 and stride == 1 and ph == 0 and pw == 0
    if bn_reduce is not None:
        by, bgam, bbeta, bsave, bscr = bn_reduce[:5]
        bmask = bn_reduce[5] if len(bn_reduce) > 5 else None
        if (add is not None or bmask is not None) and not one_by_one:
            raise ValueError("bn_reduce with add or a bit mask needs a 1x1 stride-1 data gradient (linear rows)")
        if tuple(by.shape) != (N, Cin, H, W) or bscr.shape != (2, Cin):
            raise ValueError("bn_reduce: y / scratch do not match dx")
        if bmask is not None and (bmask.dtype != torch.uint8 or bmask.numel() != N * H * W * (Cin // 8)):
            raise ValueError("bn_reduce: expected a uint8 [N*H*W, Cin/8] bit mask")
        _check_act(by, "bn_reduce.y")
        bnr = dict(bnr_y=by.data_ptr(), bnr_gamma=bgam.data_ptr(), bnr_beta=bbeta.data_ptr(),
                   bnr_mean=bsave[0].data_ptr(), bnr_invstd=bsave[1].data_ptr(), bnr_mask=_ptr(bmask))
        s1, s2 = bscr[1].data_ptr(), bscr[0].data_ptr()      # scratch layout of bn_act_bwd: [0] = dgamma, [1] = dbeta
    from . import fp8 as _fp8

    if _fp8.dgrad_eligible(Cin, Cout, R * S if stride == 1 else max(1, (R * S) // 4)) and bn_reduce is None \
            and N * H * W >= 2048 and \
            (one_by_one or (stride == 1 and USE_TILE_TMA) or s2_tile):
        # e5m2 output gradients x e4m3 weights, both K-major: the weights come as this step's transposed e4m3 copy
        # [Cin][R*S*Cout] (same scale as the forward's copy); k-blocks of 128 output channels; the epilogue (incl. the
        # shortcut-gradient add) runs on the de-quantised fp32 accumulator
        tw_ = _fp8.twin_of(dy)                      # produced by the BN-backward kernel that wrote dy, if any
        if tw_ is None:
            _fp8.request_twin(dy)
        dyq, sd = tw_ if tw_ is not None else _fp8.quantize(dy, ("dy", wp, N, P, Q), e5m2=True)
        wt, sw = _fp8.quantize_weight_t(w_bf16, R * S, Cin)
        wtp, wtr, wtc = wt.data_ptr(), Cin, R * S * Cout
        cch8 = Cout // 128
        fp8kw = dict(fp8=2, deq_a=_fp8.inv_scale_ptr(sd, dy.device), deq_b=_fp8.inv_scale_ptr(sw, dy.device))
        _fp8.count("dgrad")
        if one_by_one:
            cands = conv_variants(n_total, N * H * W, cch8, True, fp8=True)
            _tuned(("dgrad1x1_f8", N, H, W, Cin, Cout, add is not None, add_mask is not None), cands,
                   lambda v: C.conv_gemm(C.CONV_GEMM_DGRAD, 0, dx.data_ptr(), _ptr(add), 0, 0, 0, N * H * W, cch8, Cin, P,
                                         Q, Cout, H, W, 1, 1, 1, 0, 1, cch8, 0, Cin, wtp, wtr, wtc, n_total,
                                         dyq.data_ptr(), Cout, N, 0, 0, 0, 0, _stream(), 0, Cout, _ptr(add_mask), variant=v,
                                         **fp8kw))
        elif stride == 1:
            tw, th, tn = tile_geometry(H, W, N, 128)
            cands = conv_variants(n_total, N * H * W, R * S * cch8, True, fp8=True)
            _tuned(("dgrad_f8", N, H, W, Cin, Cout, R, S, ph, pw, dil, add is not None, add_mask is not None), cands,
                   lambda v: C.conv_gemm(C.CONV_TILE_DGRAD, 0, dx.data_ptr(), _ptr(add), 0, 0, 0, N * H * W,
                                         R * S * cch8, Cin, P, Q, Cout, H, W, R, S, 1, ph, dil, cch8, 0, Cin,
                                         wtp, wtr, wtc, n_total, dyq.data_ptr(), Cout, N, tw, th, tn, 0,
                                         _stream(), pw, Cout, _ptr(add_mask), variant=v, **fp8kw))
        else:
            tw, th, tn = tile_geometry((H + 1) // 2, (W + 1) // 2, N, 128)
            cands = conv_variants(n_total, N * ((H + 1) // 2) * ((W + 1) // 2),
                                              max(1, (R * S * cch8) // 4), True, fp8=True)
            _tuned(("dgrad_s2_f8", N, H, W, Cin, Cout, R, S, ph, pw, dil, zfill), cands,
                   lambda v: C.conv_gemm(C.CONV_TILE_DGRAD, 0, dx.data_ptr(), 0, 0, 0, 0, N * H * W, R * S * cch8, Cin, P,
                                         Q, Cout, H, W, R, S, 2, ph, dil, cch8, 0, Cin, wtp, wtr, wtc, n_total,
                                         dyq.data_ptr(), Cout, N, tw, th, tn, zfill, _stream(), pw, Cout, 0, variant=v,
                                         **fp8kw))
        return dx
    if R == 1 and S == 1 and stride == 1 and ph == 0 and pw == 0:
        _tuned(("dgrad1x1", N, H, W, Cin, Cout, add is not None, add_mask is not None,
                0 if bn_reduce is None else len(bn_reduce)),
               conv_variants(n_total, N * H * W, cch, True),
               lambda v: C.conv_gemm(C.CONV_GEMM_DGRAD, 0, dx.data_ptr(), _ptr(add), 0, s1, s2, N * H * W, cch, Cin, P, Q,
                                     Cout, H, W, 1, 1, 1, 0, 1, cch, 0, Cin, wp, wr, wc, n_total, dy.data_ptr(), Cout, N,
                                     0, 0, 0, 0, _stream(), 0, 0, _ptr(add_mask), variant=v, **bnr),
               (bn_reduce[4],) if bn_reduce is not None else ())
    elif stride == 1 and USE_TILE_TMA:
        tw, th, tn = tile_geometry(H, W, N, 128)
        _tuned(("dgrad", N, H, W, Cin, Cout, R, S, 1, ph, pw, dil, add is not None, add_mask is not None,
                bn_reduce is not None), conv_variants(n_total, N * H * W, R * S * cch, True),
               lambda v: C.conv_gemm(C.CONV_TILE_DGRAD, 0, dx.data_ptr(), _ptr(add), 0, s1, s2, N * H * W, R * S * cch,
                                     Cin, P, Q, Cout, H, W, R, S, 1, ph, dil, cch, 0, Cin, wp, wr, wc, n_total,
                                     dy.data_ptr(), Cout, N, tw, th, tn, 0, _stream(), pw, 0, _ptr(add_mask), variant=v,
                                     **bnr),
               (bn_reduce[4],) if bn_reduce is not None else ())
    elif s2_tile:
        # four stride-1 phase problems (one launch each), tiles iterate the half-resolution phase grid
        tw, th, tn = tile_geometry((H + 1) // 2, (W + 1) // 2, N, 128)
        _tuned(("dgrad_s2", N, H, W, Cin, Cout, R, S, 2, ph, pw, dil, zfill, bn_reduce is not None),
               conv_variants(n_total, N * ((H + 1) // 2) * ((W + 1) // 2), max(1, (R * S * cch) // 4), True),
               lambda v: C.conv_gemm(C.CONV_TILE_DGRAD, 0, dx.data_ptr(), 0, 0, s1, s2, N * H * W, R * S * cch, Cin, P,
                                     Q, Cout, H, W, R, S, 2, ph, dil, cch, 0, Cin, wp, wr, wc, n_total, dy.data_ptr(),
                                     Cout, N, tw, th, tn, zfill, _stream(), pw, 0, 0, variant=v, **bnr),
               (bn_reduce[4],) if bn_reduce is not None else ())
    else:
        C.conv_gemm(C.CONV_DGRAD, dy.data_ptr(), dx.data_ptr(), _ptr(add), 0, s1, s2, N * H * W, R * S * cch,
                    Cin, P, Q, Cout, H, W, R, S, stride, ph, dil, cch, 0, Cin, wp, wr, wc, n_total, 0, 0, N, 0, 0, 0, 0,
                    _stream(), pw, 0, _ptr(add_mask), **bnr)
    return dx


def _wgrad_splits(tiles: int, total_kb: int, device_index: int) -> int:
    target = 2 * sm_count(device_index)
    return max(1, min(total_kb, (target + tiles - 1) // tiles))


def conv_wgrad(x: torch.Tensor, dy: torch.Tensor, grad_w: torch.Tensor, kernel: Tuple[int, int], stride: int,
               pad, dil: int = 1, prepadded: Optional[torch.Tensor] = None, groups: int = 1) -> None:
    """grad_w[Cout][R*S*Cin] (fp32, KRSC) += dy^T * im2col(x).  ``prepadded``: see :func:`stem_prepare`.
    ``groups`` > 1: grad_w is the compact [Cout][R*S*Cin/groups] gradient of the grouped weight."""
    C = _C()
    _check_act(x)
    _check_act(dy, "dy")
    N, Cin, H, W = x.shape
    _, Cout, P, Q = dy.shape
    R, S = kernel
    ph, pw = _pad2(pad)
    M = N * P * Q
    dev = x.device.index or 0
    if grad_w.dtype != torch.float32:
        raise TypeError("grad_w must be fp32")
    if groups > 1:
        # tiles of 64 output channels of a bundle x (tap, the bundle's 64 T input channels); the epilogue adds the
        # in-group entries
        if not grouped_conv_native(Cin, Cout, groups):
            raise ValueError(f"grouped conv {Cin} -> {Cout} in {groups} groups is not supported by the native kernels")
        cg = Cin // groups
        if grad_w.numel() != Cout * R * S * cg:
            raise ValueError("conv_wgrad: grad_w does not match the grouped weight [Cout, Cin/groups, R, S]")
        wb, t = grouped_bundle(cg)
        ncols = R * S * t * 64
        if USE_TILE_TMA and (stride == 1 or (stride == 2 and USE_TILE_S2)):
            mode, (tw, th, tn) = C.CONV_TILE_FWD, tile_geometry(P, Q, N, 64)
            total_kb = -(-Q // tw) * -(-P // th) * -(-N // tn)
        else:
            mode, (tw, th, tn), total_kb = C.CONV_FWD, (0, 0, 0), (M + 63) // 64
        splits = _wgrad_splits(((ncols + 127) // 128) * (_ceil_div(Cout, wb) * t), total_kb, dev)
        C.conv_wgrad(mode, x.data_ptr(), dy.data_ptr(), grad_w.data_ptr(), M, Cout, Cout, R * S * cg, ncols, H, W, Cin,
                     P, Q, R, S, stride, ph, dil, 0, splits, N, tw, th, tn, _stream(), pw, t * 64, cg, group_width=cg)
        return
    if Cin <= 4:
        SP, RPK, KB, RP = stem_geometry(R, S)
        ncols = KB * 64
        scratch = torch.zeros((Cout, ncols), dtype=torch.float32, device=x.device)
        tiles = ((ncols + 127) // 128) * ((Cout + 127) // 128)
        geo = stem_tma_geometry(H, W, kernel, stride, (ph, pw)) if dil == 1 else None
        if geo is not None:
            xp = prepadded if prepadded is not None else pad_image(x, geo[0], geo[1], ph, pw, geo[2])
            tw, th, tn = tile_geometry(P, Q, N, 64)
            total_kb = -(-Q // tw) * -(-P // th) * -(-N // tn)
            C.conv_wgrad(C.CONV_STEM_TMA, xp.data_ptr(), dy.data_ptr(), scratch.data_ptr(), M, Cout, Cout, ncols, ncols,
                         geo[0], geo[1], 4, P, Q, R, S, stride, 0, 1, SP, _wgrad_splits(tiles, total_kb, dev), N, tw, th,
                         tn, _stream(), 0, 0, 0)
        else:
            C.conv_wgrad(C.CONV_STEM, x.data_ptr(), dy.data_ptr(), scratch.data_ptr(), M, Cout, Cout, ncols, ncols, H,
                         W, 4, P, Q, R, S, stride, ph, dil, SP, _wgrad_splits(tiles, (M + 63) // 64, dev), N, 0, 0, 0,
                         _stream(), pw, 0, 0)
        # grad_w is KRSC with the TRUE channel count (3): fold the packed scratch back
        cin_true = grad_w.shape[1]
        C.unpack_stem_grad(scratch.data_ptr(), grad_w.data_ptr(), Cout, R, S, cin_true, RP, SP, _stream())
        return
    if Cin % 8 != 0 or Cout % 8 != 0:
        raise ValueError("conv_wgrad needs Cin, Cout multiples of 8")
    ldw = R * S * Cin
    if R == 1 and S == 1 and stride == 1 and ph == 0 and pw == 0:
        mode, (tw, th, tn), total_kb = C.CONV_GEMM, (0, 0, 0), (M + 63) // 64
        cpad, ncols = Cin, Cin                       # one tap: virtual columns = real columns
    else:
        cpad = _ceil_div(Cin, 64) * 64
        ncols = R * S * cpad
        if USE_TILE_TMA and (stride == 1 or (stride == 2 and USE_TILE_S2)):
            mode, (tw, th, tn) = C.CONV_TILE_FWD, tile_geometry(P, Q, N, 64)
            total_kb = -(-Q // tw) * -(-P // th) * -(-N // tn)
        else:
            mode, (tw, th, tn), total_kb = C.CONV_FWD, (0, 0, 0), (M + 63) // 64
    co_tiles = _ceil_div(Cout, 64) if 0 < Cout % 128 <= 64 else _ceil_div(Cout, 128)   # narrow tail: role-swapped tiles
    tiles = ((ncols + 127) // 128) * co_tiles
    splits = _wgrad_splits(tiles, total_kb, dev)
    C.conv_wgrad(mode, x.data_ptr(), dy.data_ptr(), grad_w.data_ptr(), M, Cout, Cout, ldw, ncols, H, W, Cin, P, Q,
                 R, S, stride, ph, dil, 0, splits, N, tw, th, tn, _stream(), pw, cpad, Cin)


# ------------------------------------------------------------------------------------------------
# linear (FC) = 1x1 conv on [B, K]
# ------------------------------------------------------------------------------------------------
def linear_fwd(x: torch.Tensor, w_bf16: torch.Tensor, bias: Optional[torch.Tensor], relu: bool = False):
    """x [B, K] bf16, w [Nout, K] bf16 -> y [B, Npad] bf16 (Npad = Nout rounded up to 64; pad cols = 0)."""
    C = _C()
    _check_act(x)
    B, K = x.shape
    Nout = w_bf16.shape[0]
    if K % 8 != 0:
        raise ValueError("linear: in_features must be a multiple of 8")
    Npad = (Nout + 63) // 64 * 64
    y = torch.empty((B, Npad), dtype=torch.bfloat16, device=x.device)
    kb = _ceil_div(K, 64)
    # pad columns [Nout, Npad) are written as exact zeros (their weight rows are TMA out-of-bounds, bias is masked)
    C.conv_gemm(C.CONV_GEMM, 0, y.data_ptr(), 0, _ptr(bias), 0, 0, B, kb, Npad, 1, 1, K, 1, 1, 1, 1, 1, 0, 1,
                kb, int(relu), Nout, w_bf16.data_ptr(), Nout, K, Npad, x.data_ptr(), K, B, 0, 0, 0, 0, _stream())
    return y


def linear_dgrad(dy: torch.Tensor, w_bf16: torch.Tensor) -> torch.Tensor:
    """dy [B, Npad] bf16, w [Nout, K] -> dx [B, K].  K need not be a multiple of 64 (a squeeze-excitation fc2 has
    C/4 inputs): the N tiles cover K rounded up to 64 and the stores stop at K, as in ``conv_dgrad``."""
    C = _C()
    B, Npad = dy.shape
    Nout, K = w_bf16.shape
    dx = torch.empty((B, K), dtype=torch.bfloat16, device=dy.device)
    C.conv_gemm(C.CONV_GEMM_DGRAD, 0, dx.data_ptr(), 0, 0, 0, 0, B, Npad // 64, K, 1, 1, Npad, 1, 1, 1, 1, 1, 0,
                1, Npad // 64, 0, K, w_bf16.data_ptr(), Nout, K, _ceil_div(K, 64) * 64, dy.data_ptr(), Npad, B, 0, 0, 0, 0,
                _stream())
    return dx


def linear_wgrad(x: torch.Tensor, dy: torch.Tensor, grad_w: torch.Tensor) -> None:
    """grad_w [Nout, K] fp32 += dy[:, :Nout]^T x."""
    C = _C()
    B, K = x.shape
    Nout = grad_w.shape[0]
    Npad = dy.shape[1]
    tiles = ((K + 127) // 128) * ((Nout + 127) // 128)
    splits = _wgrad_splits(tiles, (B + 63) // 64, x.device.index or 0)
    C.conv_wgrad(C.CONV_GEMM, x.data_ptr(), dy.data_ptr(), grad_w.data_ptr(), B, Nout, Npad, K, K, 1, 1, K, 1, 1, 1,
                 1, 1, 0, 1, 0, splits, B, 0, 0, 0, _stream())


# ------------------------------------------------------------------------------------------------
# BatchNorm + activation
# ------------------------------------------------------------------------------------------------
def bn_supported(c: int) -> bool:
    """Any channel count that is a multiple of 8 (power-of-two widths take the flat thread mapping, the rest the
    64-channel-chunk mapping; see csrc/ops/bn_act.cu)."""
    return c > 0 and c % 8 == 0


def bn_act_fwd(y: torch.Tensor, stats: Optional[torch.Tensor], gamma, beta, running_mean, running_var,
               eps: float, momentum: float, relu: bool, residual: Optional[torch.Tensor], train: bool,
               want_mask: bool = False, sample_scale: Optional[torch.Tensor] = None):
    """z = act(BN(y) [+ residual]).  Returns (z, save) — with ``want_mask`` (train + ReLU) (z, save, mask): one bit per
    element telling whether z > 0, which lets the backward of residual layers skip reading z (16x less mask traffic).
    ``relu``: False / True, 2 for ReLU6 (clamp to [0, 6]; not with ``want_mask``) or 3 for hardswish
    (x * clamp(x + 3, 0, 6) / 6; not with ``want_mask`` or ``residual``), 4 for SiLU (x * sigmoid(x); the same
    refusals), 5 for GELU (x * Phi(x), erf form; the same refusals), 6 for SiLU before a ``residual`` (required):
    z = silu(BN(y)) [* sample_scale[n]] + residual (no bit mask).  ``sample_scale``: fp32 [N] (stochastic depth, train
    only): z = BN(y) * sample_scale[n] + residual, with no activation, or with code 6 as above."""
    C = _C()
    _check_act(y, "y")
    if int(relu) in (4, 5) and (want_mask or residual is not None):
        raise ValueError("bn_act_fwd: SiLU / GELU take no residual and have no bit-mask variant")
    if int(relu) == 6 and (want_mask or residual is None):
        raise ValueError("bn_act_fwd: SiLU before the residual (6) needs a residual and has no bit-mask variant")
    _check_sample_scale(sample_scale, y, relu, residual, train)
    if int(relu) == 2 and want_mask:
        raise ValueError("bn_act_fwd: ReLU6 has no bit-mask variant")
    if int(relu) == 3 and (want_mask or residual is not None):
        raise ValueError("bn_act_fwd: hardswish takes no residual and has no bit-mask variant")
    N, Ch, H, W = y.shape
    M = N * H * W
    z = torch.empty_like(y)
    if train:
        if stats is None:
            stats = zeros_f32((2, Ch), y.device)
            C.channel_stats(y.data_ptr(), stats[0].data_ptr(), stats[1].data_ptr(), M, Ch, sm_count(y.device.index or 0),
                            _stream())
        save = torch.empty((2, Ch), dtype=torch.float32, device=y.device)
        mask = torch.empty((M, Ch // 8), dtype=torch.uint8, device=y.device) if (want_mask and relu) else None
        from . import fp8 as _fp8

        zq = slot = None
        key = ("act", gamma.data_ptr(), N, H, W)
        # emit the e4m3 twin only when an fp8 convolution consumed this layer's output in an earlier step
        twin = _fp8.enabled() and int(relu) not in (2, 3, 4, 5, 6) and sample_scale is None and Ch % 128 == 0 \
            and M >= 2048 and _fp8.note_producer(z, key)
        if twin:
            idx, fused = _fp8.producer_slot(key, y.device, z)
            if fused:       # the e4m3 twin rides in this kernel's pass (+1 B/element) instead of a 3 B/element pass
                zq, slot = torch.empty_like(z, dtype=torch.uint8), _fp8.slot_ptr(idx, y.device)
        C.bn_act_fwd(y.data_ptr(), _ptr(residual), z.data_ptr(), stats[0].data_ptr(), stats[1].data_ptr(),
                     gamma.data_ptr(), beta.data_ptr(), save[0].data_ptr(), save[1].data_ptr(), _ptr(running_mean),
                     _ptr(running_var), eps, momentum, M, Ch, int(relu), True, sm_count(y.device.index or 0), _stream(),
                     _ptr(mask), _ptr(zq), slot or 0, _ptr(sample_scale), H * W)
        if twin:
            if zq is not None:
                _fp8.attach_twin(z, zq, idx)
            else:
                _fp8.attach_by_quantize(z, key)          # first sight of this layer: calibrate, then quantise
        return (z, save, mask) if want_mask else (z, save)
    C.bn_act_fwd(y.data_ptr(), _ptr(residual), z.data_ptr(), 0, 0, gamma.data_ptr(), beta.data_ptr(), 0, 0,
                 running_mean.data_ptr(), running_var.data_ptr(), eps, momentum, M, Ch, int(relu), False,
                 sm_count(y.device.index or 0), _stream(), 0)
    return (z, None, None) if want_mask else (z, None)


def _check_sample_scale(sample_scale, y, relu, residual, train) -> None:
    if sample_scale is None:
        return
    if int(relu) not in (0, 6) or residual is None or not train:
        raise ValueError("bn: a per-sample scale (stochastic depth) needs training, a residual and no activation "
                         "(or SiLU before the residual, 6)")
    if sample_scale.dtype != torch.float32 or not sample_scale.is_cuda or sample_scale.dim() != 1 \
            or sample_scale.shape[0] != y.shape[0] or not sample_scale.is_contiguous():
        raise ValueError(f"bn: sample_scale must be a contiguous CUDA fp32 [{y.shape[0]}] tensor")


def bn_act_bwd(dz: torch.Tensor, z: Optional[torch.Tensor], y: torch.Tensor, save: torch.Tensor, gamma: torch.Tensor,
               relu: bool, want_dres: bool, gamma_grad: Optional[torch.Tensor], beta_grad: Optional[torch.Tensor],
               beta: Optional[torch.Tensor] = None, had_residual: bool = True, zmask: Optional[torch.Tensor] = None,
               pre_reduced: Optional[torch.Tensor] = None, sample_scale: Optional[torch.Tensor] = None):
    """Returns (dy, dres|None, scratch); accumulates into gamma_grad / beta_grad (fp32) when given.
    ``pre_reduced``: fp32 [2, C] holding (dbeta, dgamma) already (``conv_dgrad(..., bn_reduce=...)``): only the
    elementwise pass runs.

    ReLU mask source: recomputed from y when the layer had no residual (``beta`` given), else the bit mask written by
    the forward (``zmask``), else the saved output ``z``.  ``sample_scale``: the forward's per-sample scale (stochastic
    depth): the BN sees dz * sample_scale[n] while dres = dz.  ``relu`` 6 (SiLU before the residual): the SiLU's input
    is recomputed from y (``beta`` required, ``had_residual`` ignored) and sees dz [* sample_scale[n]]; the residual's
    gradient is dz itself, returned as dres without a copy."""
    C = _C()
    _check_act(dz, "dz")
    if sample_scale is not None:
        _check_sample_scale(sample_scale, y, relu, True, True)
        if pre_reduced is not None or zmask is not None:
            raise ValueError("bn_act_bwd: a per-sample scale takes neither pre-reduced sums nor a bit mask")
    if int(relu) == 6 and (beta is None or zmask is not None or pre_reduced is not None):
        raise ValueError("bn_act_bwd: SiLU before the residual (6) recomputes its input from y (pass beta) and takes "
                         "neither a bit mask nor pre-reduced sums")
    N, Ch, H, W = y.shape
    M = N * H * W
    dy = torch.empty_like(y)
    dres = torch.empty_like(y) if (want_dres and int(relu) != 6) else None
    scratch = pre_reduced if pre_reduced is not None else zeros_f32((2, Ch), y.device)
    mask_from_x = bool(relu and beta is not None and (not had_residual or int(relu) == 6))   # z is then never read
    if pre_reduced is not None and not (mask_from_x or (relu and zmask is not None)):
        raise ValueError("pre_reduced sums are only defined for BN+ReLU layers (mask from y or from the bit mask)")
    if relu and not mask_from_x and zmask is None and z is None:
        raise ValueError("bn_act_bwd: need z or zmask for the ReLU mask of a residual layer")
    if int(relu) == 2 and not mask_from_x and zmask is not None:
        raise ValueError("bn_act_bwd: ReLU6 has no bit-mask variant (pass z)")
    if int(relu) in (3, 4, 5) and (not mask_from_x or want_dres):
        raise ValueError("bn_act_bwd: hardswish / SiLU / GELU recompute their input from y (pass beta, "
                         "had_residual=False)")
    from . import fp8 as _fp8

    dyq = slot = None
    key = ("grad", gamma.data_ptr(), N, H, W)
    twin = _fp8.enabled() and int(relu) not in (2, 3, 4, 5, 6) and sample_scale is None and Ch % 128 == 0 \
        and M >= 2048 and _fp8.note_producer(dy, key)             # an fp8 dgrad consumed it before
    if twin:
        idx, fused = _fp8.producer_slot(key, y.device, dy, e5m2=True)
        if fused:
            dyq, slot = torch.empty_like(dy, dtype=torch.uint8), _fp8.slot_ptr(idx, y.device)
    C.bn_act_bwd(dz.data_ptr(), _ptr(z), y.data_ptr(), dy.data_ptr(), _ptr(dres), save[0].data_ptr(),
                 save[1].data_ptr(), gamma.data_ptr(), _ptr(beta), scratch[0].data_ptr(), scratch[1].data_ptr(),
                 _ptr(gamma_grad), _ptr(beta_grad), M, Ch, int(relu), int(mask_from_x), sm_count(y.device.index or 0),
                 _stream(), _ptr(zmask) if (relu and not mask_from_x) else 0, pre_reduced is not None, _ptr(dyq),
                 slot or 0, _ptr(sample_scale), H * W)
    if twin:
        if dyq is not None:
            _fp8.attach_twin(dy, dyq, idx)
        else:
            _fp8.attach_by_quantize(dy, key, e5m2=True)
    if want_dres and int(relu) == 6:
        dres = dz
    return dy, dres, scratch


# ------------------------------------------------------------------------------------------------
# stem fusion: BN(train) + ReLU + max-pool on a raw conv output, and its backward
# ------------------------------------------------------------------------------------------------
def bn_relu_maxpool_fwd(y: torch.Tensor, stats: torch.Tensor, gamma, beta, running_mean, running_var, eps: float,
                        momentum: float, k: int, stride: int, pad: int):
    """pooled = maxpool(relu(BN_train(y))) without materialising the BN output.  Returns (pooled, argmax, save)."""
    C = _C()
    _check_act(y, "y")
    N, Ch, H, W = y.shape
    P, Q = _pool_out(H, k, stride, pad, False), _pool_out(W, k, stride, pad, False)
    pooled = empty_act(N, Ch, P, Q, y.device)
    arg = torch.empty((N, P, Q, Ch), dtype=torch.uint8, device=y.device)
    save = torch.empty((2, Ch), dtype=torch.float32, device=y.device)
    C.bn_relu_maxpool_fwd(y.data_ptr(), pooled.data_ptr(), arg.data_ptr(), stats[0].data_ptr(), stats[1].data_ptr(),
                          gamma.data_ptr(), beta.data_ptr(), save[0].data_ptr(), save[1].data_ptr(), _ptr(running_mean),
                          _ptr(running_var), eps, momentum, N, H, W, Ch, P, Q, k, stride, pad, sm_count(y.device.index or 0),
                          _stream())
    return pooled, arg, save


def bn_pool_bwd(dy_pooled: torch.Tensor, arg: torch.Tensor, y: torch.Tensor, save: torch.Tensor, gamma, beta,
                gamma_grad: Optional[torch.Tensor], beta_grad: Optional[torch.Tensor], k: int, stride: int, pad: int):
    """Gradient wrt the raw conv output y of maxpool(relu(BN(y))) given the pooled gradient (2 kernels: reduce, apply)."""
    C = _C()
    _check_act(dy_pooled, "dy_pooled")
    N, Ch, H, W = y.shape
    P, Q = dy_pooled.shape[2], dy_pooled.shape[3]
    dy = torch.empty_like(y)
    scratch = zeros_f32((2, Ch), y.device)
    C.bn_pool_bwd(dy_pooled.data_ptr(), arg.data_ptr(), y.data_ptr(), dy.data_ptr(), save[0].data_ptr(), save[1].data_ptr(),
                  gamma.data_ptr(), beta.data_ptr(), scratch[1].data_ptr(), scratch[0].data_ptr(), _ptr(gamma_grad),
                  _ptr(beta_grad), N, H, W, Ch, P, Q, k, stride, pad, sm_count(y.device.index or 0), _stream())
    return dy


# ------------------------------------------------------------------------------------------------
# pooling
# ------------------------------------------------------------------------------------------------
def maxpool_fwd(x: torch.Tensor, k: int, stride: int, pad: int, ceil_mode: bool = False):
    C = _C()
    _check_act(x)
    N, Ch, H, W = x.shape
    P, Q = _pool_out(H, k, stride, pad, ceil_mode), _pool_out(W, k, stride, pad, ceil_mode)
    y = empty_act(N, Ch, P, Q, x.device)
    arg = torch.empty((N, P, Q, Ch), dtype=torch.uint8, device=x.device)
    C.maxpool_fwd(x.data_ptr(), y.data_ptr(), arg.data_ptr(), N, H, W, Ch, P, Q, k, stride, pad, _stream())
    return y, arg


def maxpool_bwd(dy: torch.Tensor, arg: torch.Tensor, x_shape, k: int, stride: int, pad: int) -> torch.Tensor:
    C = _C()
    N, Ch, H, W = x_shape
    P, Q = dy.shape[2], dy.shape[3]
    dx = empty_act(N, Ch, H, W, dy.device)
    C.maxpool_bwd(dy.data_ptr(), arg.data_ptr(), dx.data_ptr(), N, H, W, Ch, P, Q, k, stride, pad, _stream())
    return dx


def _pool_out(h: int, k: int, stride: int, pad: int, ceil_mode: bool) -> int:
    if ceil_mode:
        o = -(-(h + 2 * pad - k) // stride) + 1
        if (o - 1) * stride >= h + pad:
            o -= 1
        return o
    return (h + 2 * pad - k) // stride + 1


def avgpool_fwd(x: torch.Tensor, k: int, stride: int, pad: int, count_include_pad: bool = True) -> torch.Tensor:
    C = _C()
    _check_act(x)
    N, Ch, H, W = x.shape
    P, Q = _pool_out(H, k, stride, pad, False), _pool_out(W, k, stride, pad, False)
    y = empty_act(N, Ch, P, Q, x.device)
    C.avgpool_fwd(x.data_ptr(), y.data_ptr(), N, H, W, Ch, P, Q, k, stride, pad, int(count_include_pad), _stream())
    return y


def avgpool_bwd(dy: torch.Tensor, x_shape, k: int, stride: int, pad: int, count_include_pad: bool = True):
    C = _C()
    N, Ch, H, W = x_shape
    dx = empty_act(N, Ch, H, W, dy.device)
    C.avgpool_bwd(dy.data_ptr(), dx.data_ptr(), N, H, W, Ch, dy.shape[2], dy.shape[3], k, stride, pad,
                  int(count_include_pad), _stream())
    return dx


def global_avgpool_fwd(x: torch.Tensor) -> torch.Tensor:
    C = _C()
    _check_act(x)
    N, Ch, H, W = x.shape
    y = torch.empty((N, Ch), dtype=torch.bfloat16, device=x.device)
    C.global_avgpool_fwd(x.data_ptr(), y.data_ptr(), N, H * W, Ch, _stream())
    return y


def global_avgpool_bwd(dy: torch.Tensor, x_shape) -> torch.Tensor:
    C = _C()
    N, Ch, H, W = x_shape
    dx = empty_act(N, Ch, H, W, dy.device)
    C.global_avgpool_bwd(dy.contiguous().data_ptr(), dx.data_ptr(), N, H * W, Ch, _stream())
    return dx


# ------------------------------------------------------------------------------------------------
# loss, data, misc
# ------------------------------------------------------------------------------------------------
def softmax_xent(logits: torch.Tensor, labels: torch.Tensor, classes: int, want_grad: bool = True,
                 grad_scale: Optional[float] = None, count_correct: bool = False):
    """Returns (mean loss [fp32 scalar tensor], dlogits|None, correct[2] int32|None).

    ``logits`` may be a column slice of a wider (padded) matrix: only ``stride(1) == 1`` is required.
    ``dlogits`` has the logical shape of ``logits`` and the same row stride (pad columns are zero).
    """
    C = _C()
    if logits.dtype != torch.bfloat16 or logits.stride(1) != 1:
        raise ValueError("softmax_xent: bf16 logits with unit column stride required")
    B, ncol = logits.shape
    ld = logits.stride(0) if B > 1 else max(ncol, logits.stride(0))
    loss = torch.zeros((), dtype=torch.float32, device=logits.device)
    dlog_full = torch.empty((B, ld), dtype=torch.bfloat16, device=logits.device) if want_grad else None
    corr = torch.zeros(2, dtype=torch.int32, device=logits.device) if count_correct else None
    C.softmax_xent(logits.data_ptr(), labels.data_ptr(), _ptr(dlog_full), loss.data_ptr(), 0, _ptr(corr), 1.0 / B,
                   (1.0 / B) if grad_scale is None else grad_scale, B, classes, ld, _stream())
    dlog = dlog_full[:, :ncol] if want_grad else None
    return loss, dlog, corr


def philox_images(n: int, h: int, w: int, seed: int, offset: int = 0, device=None, c_valid: int = 3) -> torch.Tensor:
    """Synthetic normal(0,1) batch as NHWC4 bf16 (logical [N,4,H,W] channels_last; channel 3 = 0)."""
    C = _C()
    x = empty_act(n, 4, h, w, device or torch.device("cuda", torch.cuda.current_device()))
    C.philox_normal_nhwc(x.data_ptr(), n * h * w, c_valid, 4, seed, offset, _stream())
    return x


def philox_labels(n: int, classes: int, seed: int, offset: int = 0, device=None) -> torch.Tensor:
    C = _C()
    t = torch.empty(n, dtype=torch.int64, device=device or torch.device("cuda", torch.cuda.current_device()))
    C.philox_labels(t.data_ptr(), n, classes, seed, offset, _stream())
    return t


def nchw_to_nhwc4(x: torch.Tensor, mean: Optional[torch.Tensor] = None, std: Optional[torch.Tensor] = None):
    """fp32 NCHW (C<=4) -> bf16 NHWC4 with optional per-channel normalisation."""
    C = _C()
    N, Ch, H, W = x.shape
    x = x.contiguous().float()
    out = empty_act(N, 4, H, W, x.device)
    C.nchw_to_nhwc_norm(x.data_ptr(), out.data_ptr(), N, Ch, H, W, 4, _ptr(mean), _ptr(std), _stream())
    return out


def cast_bf16(src: torch.Tensor, dst: torch.Tensor) -> None:
    _C().cast_f32_bf16(src.data_ptr(), dst.data_ptr(), src.numel(), _stream())


def pack_stem_weight(w: torch.Tensor, R: int, S: int) -> torch.Tensor:
    """fp32 KRSC [Cout,Cin,R,S] channels_last -> packed bf16 [Cout, KB*64]."""
    C = _C()
    Cout, Cin = w.shape[0], w.shape[1]
    SP, RPK, KB, RP = stem_geometry(R, S)
    packed = torch.empty((Cout, KB * 64), dtype=torch.bfloat16, device=w.device)
    C.pack_stem_weight(w.data_ptr(), packed.data_ptr(), Cout, R, S, Cin, RP, SP, _stream())
    return packed


def bias_relu_bwd(dy: torch.Tensor, z: torch.Tensor, dbias: Optional[torch.Tensor], relu: bool,
                  c_valid: Optional[int] = None) -> torch.Tensor:
    """Returns masked dy (= dy when relu is False); dbias[c] += column sums for c < c_valid."""
    C = _C()
    Ch = dy.shape[1]
    M = dy.numel() // Ch
    dx = torch.empty_like(dy) if relu else dy
    C.bias_relu_bwd(dy.data_ptr(), z.data_ptr(), dx.data_ptr(), _ptr(dbias), M, Ch, Ch if c_valid is None else c_valid,
                    int(relu), sm_count(dy.device.index or 0), _stream())
    return dx


def dropout(x: torch.Tensor, p: float, seed: int, offset: int, step: Optional[torch.Tensor] = None) -> torch.Tensor:
    """Philox dropout; ``step``: optional int64 device scalar mixed into the key (advanced once per training step so a
    step replayed from a CUDA graph still draws fresh masks)."""
    y = torch.empty_like(x)
    _C().dropout(x.data_ptr(), y.data_ptr(), x.numel(), p, seed, offset, _stream(), _ptr(step))
    return y


def add(a: torch.Tensor, b: torch.Tensor) -> torch.Tensor:
    y = torch.empty_like(a)
    _C().add_bf16(a.data_ptr(), b.data_ptr(), y.data_ptr(), a.numel(), _stream())
    return y


def u8_nhwc_to_nhwc4(x_u8: torch.Tensor, mean: Optional[torch.Tensor] = None, std: Optional[torch.Tensor] = None):
    """uint8 [N, H, W, 3] (decoded image bytes) -> bf16 NHWC4 activations, normalised on the device."""
    C = _C()
    if x_u8.dtype != torch.uint8 or x_u8.dim() != 4 or x_u8.shape[3] != 3 or not x_u8.is_contiguous():
        raise ValueError("expected a contiguous uint8 [N, H, W, 3] tensor")
    N, H, W, _ = x_u8.shape
    out = empty_act(N, 4, H, W, x_u8.device)
    C.nhwc_u8_to_nhwc4(x_u8.data_ptr(), out.data_ptr(), N * H * W, _ptr(mean), _ptr(std), _stream())
    return out


def check_resized_crop_desc(desc: torch.Tensor, nbytes: int, size: int) -> None:
    """Raise ValueError unless every row of the float64 [B, 8] descriptor (offset, Hr, Wr, sy, sx, oy, ox, flip) names a
    region inside an ``nbytes`` buffer and gives every one of the ``size`` output rows and columns at least one tap."""
    if desc.dtype != torch.float64 or desc.dim() != 2 or desc.shape[1] != 8 or desc.device.type != "cpu":
        raise ValueError("resized_crop: the descriptor must be a float64 [B, 8] tensor on the host")
    if not 1 <= desc.shape[0] <= 65535 or not 1 <= size <= 4096:
        raise ValueError(f"resized_crop: batch {desc.shape[0]} or size {size} out of range")
    off, hr, wr, sy, sx, oy, ox, flip = desc.unbind(1)
    ints = torch.stack([off, hr, wr, oy, ox, flip])
    if not (torch.isfinite(desc).all() and (ints == ints.trunc()).all()):
        raise ValueError("resized_crop: non-integer or non-finite descriptor entry")
    bad = (off < 0) | (hr < 1) | (wr < 1) | (off + hr * wr * 3 > nbytes) | ~((flip == 0) | (flip == 1))
    for s, o, n in ((sy, oy, hr), (sx, ox, wr)):
        support = torch.where(s >= 1, s, torch.ones_like(s))
        last = s * (o + size - 0.5)                    # center of the last output index: its first tap must be inside
        bad |= (s <= 0) | (o < 0) | (last + support >= 2 ** 30) | ((last - support + 0.5).trunc() >= n)
    if bool(bad.any()):
        i = int(bad.nonzero()[0, 0])
        raise ValueError(f"resized_crop: descriptor {i} {desc[i].tolist()} does not fit a {nbytes}-byte buffer "
                         f"at output size {size}")


def resized_crop(data: torch.Tensor, desc: torch.Tensor, size: int, mean: torch.Tensor, std: torch.Tensor):
    """Packed uint8 regions (CUDA, 1-D) + host float64 descriptor [B, 8] -> bf16 NHWC4 [B, size, size] activations:
    the antialiased bilinear resized crop, flip and (v/255 - mean)/std of every image (csrc/ops/augment.cu)."""
    if data.dtype != torch.uint8 or data.dim() != 1 or not data.is_cuda or not data.is_contiguous():
        raise ValueError("resized_crop: data must be a contiguous 1-D CUDA uint8 tensor")
    for t in (mean, std):
        if t.dtype != torch.float32 or t.numel() != 3 or t.device != data.device or not t.is_contiguous():
            raise ValueError("resized_crop: mean and std must be 3 contiguous fp32 values on the data's device")
    size = int(size)
    check_resized_crop_desc(desc, data.numel(), size)
    C = _C()
    B = desc.shape[0]
    d = desc.to(data.device, non_blocking=True)
    out = empty_act(B, 4, size, size, data.device)
    C.resized_crop(data.data_ptr(), d.data_ptr(), out.data_ptr(), B, size, mean.data_ptr(), std.data_ptr(), _stream())
    return out


def dgrad_supports_add(kernel: Tuple[int, int], stride: int) -> bool:
    """Whether conv_dgrad can fold ``+ add`` into its epilogue for this geometry without leaving the fast path
    (the stride-2 phase decomposition writes each output phase from a different launch, so it cannot)."""
    return not (stride == 2 and USE_TILE_TMA and USE_TILE_S2 and kernel[0] * kernel[1] <= 16)


def dgrad_fuses_bn_reduce(kernel: Tuple[int, int], stride: int, pad) -> bool:
    """Whether ``conv_dgrad(..., bn_reduce=...)`` costs less than the plain dgrad plus the stand-alone BN-backward
    reduction pass.  Measured on H100 at the ResNet-50 shapes: yes for 1x1 stride-1 data gradients (bandwidth-bound
    GEMMs; the y tile is fetched under the MMAs), no for window convolutions, where the statistics epilogue of their many
    short tiles costs more than the reduction pass it replaces."""
    return tuple(kernel) == (1, 1) and stride == 1 and _pad2(pad) == (0, 0)


# ------------------------------------------------------------------------------------------------
# ShuffleNetV2: channel shuffle fused into the branch BatchNorm (csrc/ops/shufflenet.cu)
# ------------------------------------------------------------------------------------------------
def _sh_bn(bn) -> tuple:
    """(sum, sumsq, gamma, beta, mean, invstd, running_mean, running_var, dgamma, dbeta, gamma_grad, beta_grad, eps,
    momentum) of the binding from a dict of tensors (missing entries: none)."""
    if bn is None:
        return (0,) * 12 + (0.0, 0.0)
    keys = ("sum", "sumsq", "gamma", "beta", "mean", "invstd", "running_mean", "running_var", "dgamma", "dbeta",
            "gamma_grad", "beta_grad")
    for k in keys:
        t = bn.get(k)
        if t is not None and (t.dtype != torch.float32 or not t.is_cuda or not t.is_contiguous()):
            raise ValueError(f"shuffle: BN {k} must be a contiguous CUDA fp32 vector")
    return tuple(_ptr(bn.get(k)) for k in keys) + (float(bn.get("eps", 0.0)), float(bn.get("momentum", 0.0)))


def _sh_geometry(ab: torch.Tensor, half: int):
    _check_act(ab, "a / b")
    N, ld_ab, H, W = ab.shape
    if half <= 0 or half % 2 != 0 or ld_ab != _ceil_div(half, 8) * 8:
        raise ValueError(f"shuffle: half = {half} must be even and the branch tensors {ld_ab} = half rounded up to 8 wide")
    return N, ld_ab, H, W


def shuffle_fwd(a: torch.Tensor, b: torch.Tensor, half: int, split: bool, train: bool, bn_b: dict,
                bn_a: Optional[dict] = None):
    """s[2i] = a[i] (a bit copy; with ``bn_a``: relu(BN_a(a[i]))), s[2i+1] = relu(BN_b(b[i])) for i < ``half``.
    ``a``, ``b``: NHWC bf16 [N, p(half), H, W] with p(c) = c rounded up to 8, zero beyond ``half``.  Returns (lo, hi) =
    (s[:, :half], s[:, half:]) as two [N, p(half), H, W] tensors (``split``) or s as one [N, p(2 half), H, W] tensor,
    zero in the pad channels.  ``bn_*``: dicts of fp32 vectors: gamma, beta, running_mean, running_var, eps, momentum;
    in training also the conv epilogue's sum / sumsq and the mean / invstd outputs the backward reads."""
    N, ld, H, W = _sh_geometry(b, half)
    if tuple(a.shape) != tuple(b.shape):
        raise ValueError("shuffle_fwd: a and b must have the same shape")
    _check_act(a, "a")
    if split:
        s0, s1 = empty_act(N, ld, H, W, b.device), empty_act(N, ld, H, W, b.device)
        ld_s = ld
    else:
        ld_s = _ceil_div(2 * half, 8) * 8
        s0, s1 = empty_act(N, ld_s, H, W, b.device), None
    _C().shuffle_fwd(a.data_ptr(), b.data_ptr(), s0.data_ptr(), _ptr(s1), N * H * W, half, ld, ld_s, int(split),
                     int(bn_a is not None), int(train), _sh_bn(bn_a), _sh_bn(bn_b), sm_count(b.device.index or 0),
                     _stream())
    return (s0, s1) if split else s0


def shuffle_bwd(ds, b: torch.Tensor, half: int, bn_b: dict, a: Optional[torch.Tensor] = None,
                bn_a: Optional[dict] = None):
    """Backward of :func:`shuffle_fwd` in training: ``ds`` the gradient of s, or the pair (dlo, dhi).  Returns (da, db):
    the pass-through gradient (a bit copy) or, with ``bn_a``, the gradient of branch1's conv output ``a``, and the
    gradient of ``b``, both [N, p(half), H, W] with zero pad channels.  ``bn_*`` as in the forward plus dgamma / dbeta
    (zeroed fp32 scratch) and the optional gamma_grad / beta_grad accumulators.  Two launches: reduce, apply."""
    N, ld, H, W = _sh_geometry(b, half)
    split = isinstance(ds, (tuple, list))
    parts = list(ds) if split else [ds]
    ld_s = ld if split else _ceil_div(2 * half, 8) * 8
    for t in parts:
        _check_act(t, "ds")
        if tuple(t.shape) != (N, ld_s, H, W):
            raise ValueError(f"shuffle_bwd: gradient of shape {tuple(t.shape)}, expected {(N, ld_s, H, W)}")
    if (bn_a is None) != (a is None):
        raise ValueError("shuffle_bwd: a and bn_a go together")
    da, db = empty_act(N, ld, H, W, b.device), empty_act(N, ld, H, W, b.device)
    _C().shuffle_bwd(parts[0].data_ptr(), parts[1].data_ptr() if split else 0, _ptr(a), b.data_ptr(), da.data_ptr(),
                     db.data_ptr(), N * H * W, half, ld, ld_s, int(split), int(bn_a is not None), _sh_bn(bn_a),
                     _sh_bn(bn_b), sm_count(b.device.index or 0), _stream())
    return da, db


# ------------------------------------------------------------------------------------------------
# GoogLeNet: segmented BatchNorm + ReLU, adaptive average pooling, row transpose (csrc/ops/inception.cu)
# ------------------------------------------------------------------------------------------------
def _seg_slice(t: torch.Tensor, col: int, c: int, M: int, name: str) -> Tuple[int, int, int]:
    """(data_ptr, row pitch, column offset) of channels [col, col + c) of an NHWC bf16 activation with M rows."""
    _check_act(t, name)
    ld = t.shape[1]
    if t.numel() != M * ld or col % 8 or ld % 8 or col < 0 or col + c > ld:
        raise ValueError(f"bn_seg: {name} must hold {M} rows and channels [{col}, {col + c}) at offsets of 8, "
                         f"got {tuple(t.shape)}")
    return t.data_ptr(), ld, col


def _seg_vec(t: Optional[torch.Tensor], c: int, name: str) -> int:
    if t is None:
        return 0
    if t.dtype != torch.float32 or not t.is_cuda or not t.is_contiguous() or t.numel() != c:
        raise ValueError(f"bn_seg: {name} must be a contiguous CUDA fp32 vector of {c}")
    return t.data_ptr()


def _seg_M(t: torch.Tensor) -> int:
    return t.numel() // t.shape[1]


def bn_seg_fwd(segs, train: bool) -> None:
    """relu(BN(.)) of up to 4 channel segments in ONE launch.  ``segs``: dicts with ``x`` / ``z`` = (tensor, column
    offset) (NHWC bf16 activations of the same rows; a segment reads channels [col, col + c) of x and writes them to z),
    ``c`` (a multiple of 8), fp32 ``gamma`` / ``beta`` / ``running_mean`` / ``running_var`` vectors of c, ``eps``,
    ``momentum``; in training also the conv epilogue's ``sum`` / ``sumsq`` and the ``mean`` / ``invstd`` outputs.
    Channels of z outside the segments are not written."""
    rows, em, M = [], [], None
    for s in segs:
        c = int(s["c"])
        M = _seg_M(s["x"][0]) if M is None else M
        xp, ldx, colx = _seg_slice(s["x"][0], s["x"][1], c, M, "x")
        zp, ldz, colz = _seg_slice(s["z"][0], s["z"][1], c, M, "z")
        v = {k: _seg_vec(s.get(k), c, k) for k in ("sum", "sumsq", "gamma", "beta", "mean", "invstd", "running_mean",
                                                   "running_var")}
        if train and not all(v[k] for k in ("sum", "sumsq", "mean", "invstd")):
            raise ValueError("bn_seg_fwd: training needs sum, sumsq, mean and invstd")
        rows.append([xp, zp, 0, 0, ldx, colx, ldz, colz, 0, 0, 0, 0, c, v["sum"], v["sumsq"], v["gamma"], v["beta"],
                     v["mean"], v["invstd"], v["running_mean"], v["running_var"], 0, 0, 0, 0])
        em.append((float(s["eps"]), float(s["momentum"])))
    dev = segs[0]["x"][0].device
    _C().bn_seg_fwd(rows, em, M, int(train), sm_count(dev.index or 0), _stream())


def bn_seg_bwd(segs) -> None:
    """Backward of :func:`bn_seg_fwd` (training) in two launches: a deterministic reduce pass and the apply pass.
    ``segs``: dicts with ``dz`` / ``x`` / ``dx`` = (tensor, column offset): the output gradient, the saved pre-BN input
    and the input gradient's destination, ``c``, fp32 ``gamma`` / ``beta`` / ``mean`` / ``invstd`` and the optional
    ``gamma_grad`` / ``beta_grad`` accumulators (the ``.grad`` slots, += dgamma / dbeta)."""
    rows, em, M, chunks = [], [], None, 0
    dev = segs[0]["x"][0].device
    # this step's dgamma / dbeta of every segment (written by the reduce pass, read by the apply pass): one buffer, so
    # that no segment's slice is freed, and handed to the next segment, before the kernels run
    sums = torch.empty((2, sum(int(s["c"]) for s in segs)), dtype=torch.float32, device=dev)
    off = 0
    for s in segs:
        c = int(s["c"])
        M = _seg_M(s["x"][0]) if M is None else M
        xp, ldx, colx = _seg_slice(s["x"][0], s["x"][1], c, M, "x")
        dzp, lddz, coldz = _seg_slice(s["dz"][0], s["dz"][1], c, M, "dz")
        dxp, lddx, coldx = _seg_slice(s["dx"][0], s["dx"][1], c, M, "dx")
        v = {k: _seg_vec(s.get(k), c, k) for k in ("gamma", "beta", "mean", "invstd", "gamma_grad", "beta_grad")}
        rows.append([xp, 0, dzp, dxp, ldx, colx, 0, 0, lddz, coldz, lddx, coldx, c, 0, 0, v["gamma"], v["beta"],
                     v["mean"], v["invstd"], 0, 0, sums[0, off].data_ptr(), sums[1, off].data_ptr(), v["gamma_grad"],
                     v["beta_grad"]])
        off += c
        em.append((0.0, 0.0))
        chunks += _ceil_div(c, 64)
    C = _C()
    gx = C.bn_seg_grid_x(M, chunks, sm_count(dev.index or 0))
    partial = torch.empty(chunks * gx * 128, dtype=torch.float32, device=dev)
    done = zeros_f32((chunks,), dev)           # counters: zero bits; the kernel leaves them zero
    C.bn_seg_bwd(rows, em, M, partial.data_ptr(), done.data_ptr(), gx, _stream())


def adaptive_avgpool_fwd(x: torch.Tensor, out_hw: Tuple[int, int]) -> torch.Tensor:
    _check_act(x)
    N, Ch, H, W = x.shape
    P, Q = out_hw
    y = empty_act(N, Ch, P, Q, x.device)
    _C().adaptive_avgpool_fwd(x.data_ptr(), y.data_ptr(), N, H, W, Ch, P, Q, sm_count(x.device.index or 0), _stream())
    return y


def adaptive_avgpool_bwd(dy: torch.Tensor, x_shape) -> torch.Tensor:
    _check_act(dy, "dy")
    N, Ch, H, W = x_shape
    dx = empty_act(N, Ch, H, W, dy.device)
    _C().adaptive_avgpool_bwd(dy.data_ptr(), dx.data_ptr(), N, H, W, Ch, dy.shape[2], dy.shape[3],
                              sm_count(dy.device.index or 0), _stream())
    return dx


def transpose_rows(x: torch.Tensor, a: int, b: int) -> torch.Tensor:
    """out[n][j][i] = x[n][i][j] for a contiguous bf16 tensor of N * a * b elements, as a [N, b * a] matrix (a % 8 == 0).
    An NHWC activation [N, C, H, W] with (a, b) = (H * W, C) comes out flattened in NCHW order (``torch.flatten``);
    (a, b) = (C, H * W) is the inverse."""
    if x.dtype != torch.bfloat16 or not x.is_cuda or a % 8 != 0 or x.numel() % (a * b) != 0:
        raise ValueError("transpose_rows: expected a CUDA bf16 tensor of N * a * b elements with a % 8 == 0")
    if not (x.is_contiguous() or x.is_contiguous(memory_format=CL)):
        raise ValueError("transpose_rows: expected dense memory")
    n = x.numel() // (a * b)
    out = torch.empty((n, a * b), dtype=torch.bfloat16, device=x.device)
    _C().transpose_rows(x.data_ptr(), out.data_ptr(), n, a, b, sm_count(x.device.index or 0), _stream())
    return out


# ------------------------------------------------------------------------------------------------
# channel concatenation (Inception / DenseNet)
# ------------------------------------------------------------------------------------------------
def concat_channels(parts) -> torch.Tensor:
    """NHWC concat along channels of up to 8 tensors (channel counts multiples of 8)."""
    for t in parts:
        _check_act(t, "part")
    N, _, H, W = parts[0].shape
    chans = [int(t.shape[1]) for t in parts]
    out = empty_act(N, sum(chans), H, W, parts[0].device)
    _C().concat_channels([t.data_ptr() for t in parts], chans, out.data_ptr(), N * H * W, False, _stream())
    return out


def split_channels(whole: torch.Tensor, chans) -> list:
    """Inverse of :func:`concat_channels` (its backward): contiguous NHWC slices of ``whole``."""
    _check_act(whole, "whole")
    N, _, H, W = whole.shape
    parts = [empty_act(N, int(c), H, W, whole.device) for c in chans]
    _C().concat_channels([t.data_ptr() for t in parts], [int(c) for c in chans], whole.data_ptr(), N * H * W, True,
                         _stream())
    return parts
