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


def conv_variants(n_total: int, m_rows: int, kb: int, b_mn_major: bool, fp8: bool = False):
    """Variant words worth timing for an ``m_rows`` x ``n_total`` x ``kb*64`` problem (see launch_fwd_mode).  fp8
    operands run on the one-tile kernel only."""
    out = [VAR_ONE_TILE]
    if fp8 or m_rows < 128 * 132:     # less than one wave of 128-row tiles: the persistent kernels cannot pay
        return out
    out.append(VAR_PERSISTENT)
    if not (b_mn_major and n_total % 128 != 0):       # MN-major weight tiles split into two 64-column boxes
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


# ------------------------------------------------------------------------------------------------
# convolution forward / dgrad / wgrad
# ------------------------------------------------------------------------------------------------
def conv_fwd(x: torch.Tensor, w_bf16: torch.Tensor, kernel: Tuple[int, int], stride: int, pad, dil: int = 1,
             stats: bool = False, bias: Optional[torch.Tensor] = None, relu: bool = False,
             cout: Optional[int] = None, prepadded: Optional[torch.Tensor] = None):
    """y = conv(x, w) [+ bias][ReLU]; optionally per-channel (sum, sumsq) of y for BatchNorm.
    ``prepadded``: result of :func:`stem_prepare` for this (x, geometry) — skips the internal padding copy.

    ``w_bf16``: [Cout, R*S*Cin] bf16 (or the packed stem matrix [Cout, KB*64]); ``pad``: int or (pad_h, pad_w).
    """
    C = _C()
    _check_act(x)
    N, Cin, H, W = x.shape
    R, S = kernel
    ph, pw = _pad2(pad)
    Cout = cout if cout is not None else w_bf16.shape[0]
    if Cout % 8 != 0:
        raise ValueError("conv_fwd: Cout must be a multiple of 8")
    P, Q = conv_out_hw(H, W, kernel, stride, (ph, pw), dil)
    M = N * P * Q
    y = empty_act(N, Cout, P, Q, x.device)
    st = zeros_f32((2, Cout), x.device) if stats else None
    s_ptr, ss_ptr = (st[0].data_ptr(), st[1].data_ptr()) if stats else (0, 0)
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
               bn_reduce: Optional[tuple] = None) -> torch.Tensor:
    """dx = conv_transpose(dy, w) (+ add [gated by the bit mask ``add_mask``: uint8 [M, Cin/8]]).
    ``w_bf16`` is the forward matrix [Cout, R*S*Cin].

    ``bn_reduce = (y, gamma, beta, save, scratch)``: dx is the output gradient of a BN+ReLU layer whose saved input is
    ``y``; the kernel's epilogue then also accumulates that BN's dbeta / dgamma sums into ``scratch`` (fp32 [2, Cin],
    zeroed), so ``bn_act_bwd(..., pre_reduced=scratch)`` can skip its reduction pass over (dx, y)."""
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
    if add is not None:
        _check_act(add, "add")
    if add_mask is not None and (add is None or add_mask.dtype != torch.uint8 or add_mask.numel() != N * H * W * (Cin // 8)):
        raise ValueError("add_mask: expected a uint8 [N*H*W, Cin/8] bit mask accompanying `add`")
    n_total = _ceil_div(Cin, 64) * 64
    cch = _ceil_div(Cout, 64)
    wp, wr, wc = w_bf16.data_ptr(), w_bf16.shape[0], w_bf16.shape[1]
    bnr = {}
    s1 = s2 = 0
    if bn_reduce is not None:
        by, bgam, bbeta, bsave, bscr = bn_reduce
        if add is not None:
            raise ValueError("bn_reduce cannot be combined with add (the sums are taken before the epilogue add)")
        if tuple(by.shape) != (N, Cin, H, W) or bscr.shape != (2, Cin):
            raise ValueError("bn_reduce: y / scratch do not match dx")
        _check_act(by, "bn_reduce.y")
        bnr = dict(bnr_y=by.data_ptr(), bnr_gamma=bgam.data_ptr(), bnr_beta=bbeta.data_ptr(),
                   bnr_mean=bsave[0].data_ptr(), bnr_invstd=bsave[1].data_ptr())
        s1, s2 = bscr[1].data_ptr(), bscr[0].data_ptr()      # scratch layout of bn_act_bwd: [0] = dgamma, [1] = dbeta
    from . import fp8 as _fp8

    one_by_one = R == 1 and S == 1 and stride == 1 and ph == 0 and pw == 0
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
        _tuned(("dgrad1x1", N, H, W, Cin, Cout, add is not None, add_mask is not None, bn_reduce is not None),
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
               pad, dil: int = 1, prepadded: Optional[torch.Tensor] = None) -> None:
    """grad_w[Cout][R*S*Cin] (fp32, KRSC) += dy^T * im2col(x).  ``prepadded``: see :func:`stem_prepare`."""
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
    """dy [B, Npad] bf16, w [Nout, K] -> dx [B, K]."""
    C = _C()
    B, Npad = dy.shape
    Nout, K = w_bf16.shape
    dx = torch.empty((B, K), dtype=torch.bfloat16, device=dy.device)
    C.conv_gemm(C.CONV_GEMM_DGRAD, 0, dx.data_ptr(), 0, 0, 0, 0, B, Npad // 64, K, 1, 1, Npad, 1, 1, 1, 1, 1, 0,
                1, Npad // 64, 0, K, w_bf16.data_ptr(), Nout, K, K, dy.data_ptr(), Npad, B, 0, 0, 0, 0, _stream())
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
               want_mask: bool = False):
    """z = act(BN(y) [+ residual]).  Returns (z, save) — with ``want_mask`` (train + ReLU) (z, save, mask): one bit per
    element telling whether z > 0, which lets the backward of residual layers skip reading z (16x less mask traffic)."""
    C = _C()
    _check_act(y, "y")
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
        twin = _fp8.enabled() and Ch % 128 == 0 and M >= 2048 and _fp8.note_producer(z, key)
        if twin:
            idx, fused = _fp8.producer_slot(key, y.device, z)
            if fused:       # the e4m3 twin rides in this kernel's pass (+1 B/element) instead of a 3 B/element pass
                zq, slot = torch.empty_like(z, dtype=torch.uint8), _fp8.slot_ptr(idx, y.device)
        C.bn_act_fwd(y.data_ptr(), _ptr(residual), z.data_ptr(), stats[0].data_ptr(), stats[1].data_ptr(),
                     gamma.data_ptr(), beta.data_ptr(), save[0].data_ptr(), save[1].data_ptr(), _ptr(running_mean),
                     _ptr(running_var), eps, momentum, M, Ch, int(relu), True, sm_count(y.device.index or 0), _stream(),
                     _ptr(mask), _ptr(zq), slot or 0)
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


def bn_act_bwd(dz: torch.Tensor, z: Optional[torch.Tensor], y: torch.Tensor, save: torch.Tensor, gamma: torch.Tensor,
               relu: bool, want_dres: bool, gamma_grad: Optional[torch.Tensor], beta_grad: Optional[torch.Tensor],
               beta: Optional[torch.Tensor] = None, had_residual: bool = True, zmask: Optional[torch.Tensor] = None,
               pre_reduced: Optional[torch.Tensor] = None):
    """Returns (dy, dres|None, scratch); accumulates into gamma_grad / beta_grad (fp32) when given.
    ``pre_reduced``: fp32 [2, C] holding (dbeta, dgamma) already (``conv_dgrad(..., bn_reduce=...)``): only the
    elementwise pass runs.

    ReLU mask source: recomputed from y when the layer had no residual (``beta`` given), else the bit mask written by
    the forward (``zmask``), else the saved output ``z``."""
    C = _C()
    _check_act(dz, "dz")
    N, Ch, H, W = y.shape
    M = N * H * W
    dy = torch.empty_like(y)
    dres = torch.empty_like(y) if want_dres else None
    scratch = pre_reduced if pre_reduced is not None else zeros_f32((2, Ch), y.device)
    mask_from_x = bool(relu and beta is not None and not had_residual)     # z is not read at all in that case
    if pre_reduced is not None and not mask_from_x:
        raise ValueError("pre_reduced sums are only defined for BN+ReLU layers without residual")
    if relu and not mask_from_x and zmask is None and z is None:
        raise ValueError("bn_act_bwd: need z or zmask for the ReLU mask of a residual layer")
    from . import fp8 as _fp8

    dyq = slot = None
    key = ("grad", gamma.data_ptr(), N, H, W)
    twin = _fp8.enabled() and Ch % 128 == 0 and M >= 2048 and _fp8.note_producer(dy, key)   # an fp8 dgrad consumed it before
    if twin:
        idx, fused = _fp8.producer_slot(key, y.device, dy, e5m2=True)
        if fused:
            dyq, slot = torch.empty_like(dy, dtype=torch.uint8), _fp8.slot_ptr(idx, y.device)
    C.bn_act_bwd(dz.data_ptr(), _ptr(z), y.data_ptr(), dy.data_ptr(), _ptr(dres), save[0].data_ptr(),
                 save[1].data_ptr(), gamma.data_ptr(), _ptr(beta), scratch[0].data_ptr(), scratch[1].data_ptr(),
                 _ptr(gamma_grad), _ptr(beta_grad), M, Ch, int(relu), int(mask_from_x), sm_count(y.device.index or 0),
                 _stream(), _ptr(zmask) if (relu and not mask_from_x) else 0, pre_reduced is not None, _ptr(dyq),
                 slot or 0)
    if twin:
        if dyq is not None:
            _fp8.attach_twin(dy, dyq, idx)
        else:
            _fp8.attach_by_quantize(dy, key, e5m2=True)
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


def dgrad_supports_add(kernel: Tuple[int, int], stride: int) -> bool:
    """Whether conv_dgrad can fold ``+ add`` into its epilogue for this geometry without leaving the fast path
    (the stride-2 phase decomposition writes each output phase from a different launch, so it cannot)."""
    return not (stride == 2 and USE_TILE_TMA and USE_TILE_S2 and kernel[0] * kernel[1] <= 16)


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
