"""C++ host runtime: bucket planner, fd channel (SURVEY.md section 4: determinism of the bucket plan)."""
import multiprocessing as mp
import os

import pytest

from distributeddeeplearning_b200 import _ext


@pytest.fixture(scope="module")
def C():
    return _ext.load()


def test_plan_is_deterministic_and_aligned(C):
    numels = [1000, 64, 64, 2048 * 1000, 10, 513, 4096]
    a = C.plan_buckets(numels, 256, 4096, 64, 2048)
    b = C.plan_buckets(numels, 256, 4096, 64, 2048)
    assert a == b and a["hash"] == b["hash"]
    for off in a["param_offset"]:
        assert off % 64 == 0
    for start, n in zip(a["bucket_start"], a["bucket_numel"]):
        assert n % 2048 == 0 and start % 2048 == 0
    # buckets tile the arena without gaps
    pos = 0
    for start, n in zip(a["bucket_start"], a["bucket_numel"]):
        assert start == pos
        pos += n
    assert pos == a["total_elems"]
    # every parameter lies inside its bucket, in order
    for i, (bk, off) in enumerate(zip(a["param_bucket"], a["param_offset"])):
        assert a["bucket_start"][bk] <= off
        assert off + numels[i] <= a["bucket_start"][bk] + a["bucket_numel"][bk]
    assert sum(a["bucket_param_count"]) == len(numels)


def test_plan_hash_changes_with_sizes(C):
    a = C.plan_buckets([100, 200, 300], 256, 4096, 64, 2048)
    b = C.plan_buckets([100, 201, 300], 256, 4096, 64, 2048)
    assert a["hash"] != b["hash"]


def test_first_bucket_is_small(C):
    a = C.plan_buckets([1 << 16] * 20, 1 << 16, 1 << 20, 64, 2048)
    assert a["bucket_param_count"][0] == 1 and a["bucket_param_count"][1] > 1


def test_plan_rejects_bad_args(C):
    with pytest.raises(Exception):
        C.plan_buckets([10], 0, 10, 64, 2048)
    with pytest.raises(Exception):
        C.plan_buckets([10], 256, 4096, 64, 100)


def _fd_worker(rank, world, session, q):
    from distributeddeeplearning_b200 import _ext

    C = _ext.load()
    # memfd + pread: several peers read the same descriptor without consuming it (like a VMM handle)
    fd = os.memfd_create(f"r{rank}")
    os.write(fd, f"hello from {rank}".encode())
    fds = C.exchange_fds(rank, world, fd, session, 20000)
    got = {}
    for src, pfd in enumerate(fds):
        if src == rank:
            assert pfd == -1
            continue
        got[src] = os.pread(pfd, 64, 0).decode()
    fd2 = os.memfd_create("root")
    os.write(fd2, b"root-payload")
    bfd = C.broadcast_fd(rank, world, 0, fd2, session + "b", 20000)
    got["bcast"] = os.pread(bfd, 64, 0).decode() if rank != 0 else "root"
    q.put((rank, got))


def test_fd_exchange_between_processes():
    ctx = mp.get_context("spawn")
    world, session = 3, f"ddltest{os.getpid()}"
    q = ctx.Queue()
    ps = [ctx.Process(target=_fd_worker, args=(r, world, session, q)) for r in range(world)]
    for p in ps:
        p.start()
    res = dict(q.get(timeout=60) for _ in range(world))
    for p in ps:
        p.join(30)
    for r in range(world):
        for src in range(world):
            if src != r:
                assert res[r][src] == f"hello from {src}"
        assert res[r]["bcast"] == ("root" if r == 0 else "root-payload")


def test_driver_probe_does_not_raise(C):
    assert C.driver_available() in (True, False)


def test_launch_accounting_table_matches_module(C):
    """Every entry of the kernel-launch accounting table names a real binding (bench.py's gpu_launches relies on it)."""
    from distributeddeeplearning_b200 import _ext

    missing = [k for k in _ext.KERNEL_LAUNCHES if not hasattr(C, k)]
    assert not missing, missing
    for hook in ("set_conv_persistent", "set_conv_cluster", "set_wgrad_swap", "set_conv_force_stages", "set_conv_wait_hint"):
        assert hasattr(C, hook), hook
    n0 = _ext.launch_count()
    _ext.add_launches(7)
    assert _ext.launch_count() == n0 + 7


def test_tile_geometry_maximises_useful_rows():
    """The TMA pixel box of the tile-mode convolutions: never more rows than the MMA tile, always covering the map, and
    at least as many useful rows as the naive full-width choice (14x14 maps: 77 % -> 96 %)."""
    import math

    from distributeddeeplearning_b200.ops import native as nv

    def eff(P, Q, N, rows, t):
        tw, th, tn = t
        return (tw * th * tn / rows) * (Q / (math.ceil(Q / tw) * tw)) * (P / (math.ceil(P / th) * th)) * \
            (N / (math.ceil(N / tn) * tn))

    for rows in (64, 128):
        for hw in (7, 8, 13, 14, 17, 28, 35, 56, 112):
            for n in (1, 2, 32, 256):
                t = nv.tile_geometry(hw, hw, n, rows)
                tw, th, tn = t
                assert 1 <= tw <= hw and 1 <= th <= hw and 1 <= tn <= n and tw * th * tn <= rows
                naive_th = max(1, min(hw, rows // hw)) if hw <= rows else 1
                naive = (hw if hw <= rows else -(-hw // -(-hw // rows)), naive_th,
                         max(1, min(n, rows // (hw * naive_th))) if (hw <= rows and naive_th == hw) else 1)
                assert eff(hw, hw, n, rows, t) >= eff(hw, hw, n, rows, naive) - 1e-9, (hw, n, rows, t, naive)
    assert eff(14, 14, 256, 128, nv.tile_geometry(14, 14, 256, 128)) > 0.95
    assert eff(7, 7, 256, 128, nv.tile_geometry(7, 7, 256, 128)) > 0.9


def test_step_launcher_accounting_without_a_gpu(C):
    """The native hook -> bucket-launch sequencer (csrc/runtime/step_launcher.cpp): plan validation, per-parameter
    accounting, the hook callable and reset — in `hold` mode, where nothing is launched (no GPU here)."""
    plan = C.plan_buckets([4096, 64, 64, 8192, 128], 2048, 8192, 64, 2048)
    ctx = C.CommCtx([0], 0, 0, 1, 0, 0, 0, 0, 0, 0, 0, 10 ** 9)
    calls = {"stream": 0, "hyper": 0}

    def stream_fn():
        calls["stream"] += 1
        return 0

    def hyper_fn(handle):
        calls["hyper"] += 1

    def make(param_bucket):
        return C.StepLauncher(param_bucket, list(plan["bucket_param_count"]), list(plan["bucket_start"]),
                              list(plan["bucket_numel"]), ctx, 1, 0, 0, 0, 0, 0, 32, 148, False, False, 0, 0, 0, 0,
                              stream_fn, hyper_fn)

    with pytest.raises(ValueError):
        make([99] * 5)                                        # bucket id out of range
    sl = make(list(plan["param_bucket"]))
    sl.set_hold(True)
    hooks = [sl.hook(i) for i in range(5)]
    assert sl.on_ready(0) == 0 and sl.on_ready(0) == 0        # second call for the same parameter is ignored
    for h in hooks[1:]:
        assert h("the parameter autograd passes in") is None  # the hook signature: hook(param)
    assert sl.next_bucket == 0 and sl.launches == 0 and calls == {"stream": 0, "hyper": 0}
    with pytest.raises(IndexError):
        sl.on_ready(5)
    sl.reset()
    assert sl.on_ready(4) == 0 and sl.launches == 0
    # the side-stream bookkeeping is module-wide: nothing noted -> nothing to join (and no CUDA call is made)
    assert C.wgrad_join(0) is False


def test_conv_variant_words_are_well_formed():
    """The autotuner's candidate list (ops/native.py) only produces variant words the launcher understands
    (conv_gemm.cu: bits 0-3 kernel 1 = one tile / 2 = persistent, bit 8 CTA pair, only with the persistent kernel) —
    never the epilogue debug bits 12-14 of tools/epi_probe.py — and the fp8 forward convolutions only the one-tile kernel."""
    from distributeddeeplearning_b200.ops import native

    seen = set()
    for n_total in (64, 128, 192, 256, 512, 1024, 2048):
        for m_rows in (128, 128 * 132 - 1, 128 * 132, 802816):
            for kb in (1, 4, 18, 36):
                for mn in (False, True):
                    cands = native.conv_variants(n_total, m_rows, kb, mn)
                    assert cands[0] == native.VAR_ONE_TILE and len(set(cands)) == len(cands)
                    if m_rows < 128 * 132:
                        assert cands == [native.VAR_ONE_TILE]
                    for v in cands:
                        assert v >> 9 == 0, hex(v)                       # nothing above the pair bit
                        kind, width, pair = v & 0xf, (v >> 4) & 0xf, (v >> 8) & 1
                        assert kind in (1, 2) and width == 0
                        if pair:
                            assert kind == 2 and (not mn or n_total % 128 == 0)   # MN-major halves: 64-column boxes
                        name = native.variant_name(v)
                        assert name.startswith(("one-tile", "persistent"))
                        seen.add(name)
                    assert native.conv_variants(n_total, m_rows, kb, mn, fp8=True) == [native.VAR_ONE_TILE]
    assert {"one-tile", "persistent", "persistent-pair"} <= seen


def test_fp8_eligibility_rules():
    """fp8 operands only where they pay and where the geometry allows (ops/fp8.py): reduction >= MIN_K elements, 128-channel
    operand rows; everything else (stem, layer1's 64-channel convs, the classifier) stays bf16."""
    from distributeddeeplearning_b200.ops import fp8

    was = fp8.enabled()
    try:
        fp8.enable(False)
        assert not fp8.fwd_eligible(512, 512, 9) and not fp8.dgrad_eligible(512, 512, 9)
        fp8.enable(True)
        assert fp8.MIN_K == 512
        assert fp8.fwd_eligible(512, 128, 1) and fp8.fwd_eligible(128, 128, 9) and fp8.fwd_eligible(1024, 2048, 1)
        assert not fp8.fwd_eligible(256, 64, 1)            # K = 256 < 512: epilogue-bound, bf16 is faster
        assert not fp8.fwd_eligible(64, 64, 9)             # 64-channel rows are not a whole fp8 k-block
        assert not fp8.fwd_eligible(3, 64, 49)             # stem
        assert fp8.dgrad_eligible(128, 512, 1) and not fp8.dgrad_eligible(64, 256, 1) and not fp8.dgrad_eligible(512, 1000, 1)
    finally:
        fp8.enable(was)
