"""The on-demand memory test on a real H100.

- The march kernel of hbm_memtest.cuh, launched directly (tests/native/libmemtest_kernels_test.so) on torch-owned
  segments and compared element by element with tests/memtest_oracle.py: checksum, mismatches, first bad word, the
  whole buffer after each element, a guard region past each segment and the control blocks' reset, at the pipeline
  edges (1-tile segments, k tiles per CTA around the stage count, more CTAs than tiles, a short last segment) and with
  faults in every lane, at segment boundaries, in the last word and as a checksum-preserving pair.
- Two segments that are two virtual mappings of one physical allocation: every reading element mismatches.
- b2dp_memtest through the ABI: exact sizing, injected faults, memory handed back, the probe ring untouched, the
  latch and its reset, the busy skip, and the daemon's -memtest_at_start.

The machines are shared: no test asks for more than 8 GiB."""
import ctypes as C
import os
import random
import signal
import subprocess
import sys
import time

import numpy as np
import pytest

import memtest_oracle as mt
from oracle import probe as oprobe

pytestmark = pytest.mark.gpu

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(HERE)
LIB_PATH = os.path.join(HERE, "native", "libmemtest_kernels_test.so")
MiB, GiB = 1 << 20, 1 << 30
U64 = C.c_uint64
GUARD_WORDS = 4096
SENTINEL = 0xA5A5A5A5


class ProbeOut(C.Structure):
    _fields_ = [("checksum", U64), ("mismatches", U64), ("first_bad", U64), ("t_start_ns", U64), ("t_end_ns", U64),
                ("seq", U64)]


class ProbeCtl(C.Structure):
    _fields_ = [("checksum", U64), ("mismatches", U64), ("first_bad", U64), ("t_start_ns", U64), ("done", C.c_uint32),
                ("pad", C.c_uint32)]


class Harness:
    def __init__(self, device=0):
        L = C.CDLL(LIB_PATH)
        L.mk_open.restype = C.c_void_p
        L.mk_open.argtypes = [C.c_int, C.c_char_p, C.c_int]
        L.mk_close.argtypes = [C.c_void_p]
        L.mk_error.restype = C.c_char_p
        L.mk_error.argtypes = [C.c_void_p]
        L.mk_sms.argtypes = [C.c_void_p]
        L.mk_element.argtypes = [C.c_void_p, C.POINTER(U64), C.POINTER(U64), C.c_int, C.c_uint32, C.c_int, C.c_int, U64,
                                 C.POINTER(ProbeOut)]
        L.mk_read_ctl.argtypes = [C.c_void_p, C.c_int, C.POINTER(ProbeCtl)]
        L.mk_occupancy.argtypes = [C.c_void_p, C.c_int, C.POINTER(C.c_int)]
        L.mk_alias_alloc.argtypes = [C.c_void_p, U64, C.POINTER(U64), C.POINTER(U64), C.POINTER(U64), C.POINTER(C.c_void_p)]
        L.mk_alias_free.argtypes = [C.c_void_p, C.c_void_p]
        self.L = L
        err = C.create_string_buffer(512)
        self.h = L.mk_open(device, err, len(err))
        if not self.h:
            raise RuntimeError("mk_open: " + err.value.decode())
        self.sms = L.mk_sms(self.h)
        self.tile_bytes = L.mk_tile_bytes()
        self.seq = 0

    def close(self):
        if self.h:
            self.L.mk_close(self.h)
            self.h = None

    def _check(self, rc, what):
        if rc == 1:
            raise RuntimeError("%s: %s" % (what, self.L.mk_error(self.h).decode()))
        assert rc == 0, "%s refused: code %d" % (what, rc)

    def element(self, ptrs, sizes, seed, elem, grid):
        self.seq += 1
        out = ProbeOut()
        n = len(ptrs)
        rc = self.L.mk_element(self.h, (U64 * n)(*ptrs), (U64 * n)(*sizes), n, seed, elem, grid, self.seq, C.byref(out))
        self._check(rc, "mk_element")
        return out

    def ctl(self, elem):
        c = ProbeCtl()
        self._check(self.L.mk_read_ctl(self.h, elem, C.byref(c)), "mk_read_ctl")
        return c

    def occupancy(self, mode):
        n = C.c_int()
        self._check(self.L.mk_occupancy(self.h, mode, C.byref(n)), "mk_occupancy")
        return n.value


@pytest.fixture(scope="module")
def H():
    if not os.path.exists(LIB_PATH):
        pytest.skip("run __graft_entry__.build() first")
    h = Harness(0)
    yield h
    h.close()


def _to_u32(t):
    return t.cpu().numpy().view(np.uint32)


def _run_case(H, seg_tiles, grid, faults, seed):
    """All four elements over segments of seg_tiles tiles each, compared with the oracle after every element."""
    import torch
    tw = H.tile_bytes // 4
    words = [k * tw for k in seg_tiles]
    segs = [torch.full((w + GUARD_WORDS,), SENTINEL - (1 << 32), dtype=torch.int32, device="cuda:0") for w in words]
    ptrs, sizes = [s.data_ptr() for s in segs], [w * 4 for w in words]
    want = mt.march(words, seed, faults)
    starts = np.cumsum([0] + words)
    for k in range(4):
        if k == 1 and faults:                            # faults are applied right after E0
            for w, mask in faults:
                g = int(np.searchsorted(starts, w, side="right") - 1)
                i = w - int(starts[g])
                v = int(segs[g][i].item()) & 0xFFFFFFFF
                v ^= mask
                segs[g][i] = v - (1 << 32) if v >= 1 << 31 else v
        r = H.element(ptrs, sizes, seed, k, grid)
        cs, mm, fb, buf = want[k]
        assert (r.checksum, r.mismatches, r.first_bad) == (cs, mm, fb), (k, seg_tiles, grid)
        got = np.concatenate([_to_u32(s)[:w] for s, w in zip(segs, words)])
        assert np.array_equal(got, buf), (k, seg_tiles, grid, np.nonzero(got != buf)[0][:8])
        for s, w in zip(segs, words):
            assert np.all(_to_u32(s)[w:] == SENTINEL), "guard region written"
        c = H.ctl(k)
        assert (c.checksum, c.mismatches, c.first_bad, c.t_start_ns, c.done) == (0, 0, (1 << 64) - 1, (1 << 64) - 1, 0)


def _cases():
    S = 3                                                # kTmaStages
    cases = [("one_tile_segments", [1, 1, 1, 1, 1], 0, [])]
    for k in (1, S - 1, S, S + 1, 2 * S - 1, 2 * S, 2 * S + 1):
        cases.append(("k%d_per_cta" % k, [5] * (4 * k // 5) + ([4 * k % 5] if 4 * k % 5 else []), 4, []))
    cases += [
        ("more_ctas_than_tiles", [4, 4, 2], 64, []),
        ("short_last_segment", [8, 8, 3], 0, []),
        ("uneven_grid", [7, 7, 7, 5], 5, []),
    ]
    tw = 4096                                           # words per 16 KiB tile
    lanes = [(4 * 1000 + lane, 1 << (lane * 7)) for lane in range(4)]
    bounds = [(8 * tw - 1, 0x80000000), (8 * tw, 0x1), (16 * tw - 1, 0xFFFFFFFF), (16 * tw, 0x00010000)]
    cases += [
        ("fault_each_lane", [8, 8, 3], 0, lanes),
        ("fault_segment_boundaries", [8, 8, 3], 0, bounds),
        ("fault_last_word", [8, 8, 3], 0, [(19 * tw - 1, 0x40)]),
        ("fault_word_zero_small_grid", [2, 2, 1], 3, [(0, 0x2)]),
    ]
    return cases


@pytest.mark.parametrize("name,seg_tiles,grid,faults", _cases(), ids=[c[0] for c in _cases()])
def test_march_kernel_matches_oracle(H, name, seg_tiles, grid, faults):
    _run_case(H, seg_tiles, grid, faults, random.Random(name).getrandbits(32))


def test_march_kernel_checksum_preserving_pair(H):
    """Two flips of one bit in opposite directions leave every checksum as it was: only the mismatch count sees them."""
    seed = 0x5EED1234
    words = [8 * 4096, 8 * 4096, 3 * 4096]
    p = mt.march(words, seed)[0][3]
    bit = 9
    a = next(i for i in range(100, 10000) if not (p[i] >> bit) & 1)
    b = next(i for i in range(30000, 40000) if (p[i] >> bit) & 1)
    faults = [(a, 1 << bit), (b, 1 << bit)]
    res = mt.march(words, seed, faults)
    clean = mt.march(words, seed)
    assert all(res[k][0] == clean[k][0] for k in (1, 2, 3)) and all(res[k][1] == 2 for k in (1, 2, 3))
    _run_case(H, [8, 8, 3], 0, faults, seed)


def test_march_kernel_keeps_two_ctas_per_sm(H):
    for mode in (0, 1, 2):
        assert H.occupancy(mode) >= 2


def test_aliased_segments_mismatch_in_every_reading_element(H):
    """Two segments that are two virtual mappings of ONE physical allocation: what E0 writes through one view, the
    other view reads under another segment seed (a data race on aliased memory, by design -- not a fault)."""
    va0, va1, size, handle = U64(), U64(), U64(), C.c_void_p()
    rc = H.L.mk_alias_alloc(H.h, 4 * MiB, C.byref(va0), C.byref(va1), C.byref(size), C.byref(handle))
    try:
        H._check(rc, "mk_alias_alloc")
        ptrs, sizes = [va0.value, va1.value], [size.value, size.value]
        H.element(ptrs, sizes, 0x1234, 0, 0)
        for k in (1, 2, 3):
            r = H.element(ptrs, sizes, 0x1234, k, 0)
            assert r.mismatches >= size.value // 4, (k, r.mismatches)
    finally:
        H.L.mk_alias_free(H.h, handle)


# ---- through the ABI --------------------------------------------------------------------------------------------------
@pytest.fixture(scope="module")
def P(pkg):
    return pkg


def _open(P, nbytes=64 * MiB):
    return P.Context("cuda:devices=0,bytes=%d,calib=1" % nbytes)


def test_memtest_clean_exact_size_and_memory_back(P):
    import torch
    torch.cuda.init()
    max_bytes = 2 * GiB + 6 * MiB
    with _open(P) as ctx:
        ctx.memtest(0, max_bytes=4 * MiB)                 # first launch loads the kernels: not counted below
        free0, _ = torch.cuda.mem_get_info(0)
        (r,) = ctx.memtest(0, max_bytes=max_bytes)
        free1, _ = torch.cuda.mem_get_info(0)
        plan = mt.plan(r.free_before, r.total_memory, 0, max_bytes)
        assert plan == [GiB, GiB, 6 * MiB]
        assert r.healthy and r.err == 0, r
        assert r.bytes_tested == sum(plan) == max_bytes and r.n_segments == 3
        assert r.mismatches == [0, 0, 0, 0] and r.first_bad_word == (1 << 64) - 1
        assert not r.flags & (P._native.MT_PARTIAL | P._native.MT_SKIPPED_BUSY | P._native.MT_ECC), r
        assert r.ms > 0 and abs(r.gbs - 6 * r.bytes_tested / r.ms * 1e-6) < 1e-3 * r.gbs
        assert abs(free1 - free0) < 2 * MiB, (free0, free1)         # every segment was freed before the call returned
        (p,) = ctx.probe_health(min_gbs=1e-3)
        assert p.healthy and not p.flags & P._native.RES_MEMTEST
    print("memtest %d bytes in %d segments: %.2f ms, %.0f GB/s" % (r.bytes_tested, r.n_segments, r.ms, r.gbs))


@pytest.mark.parametrize("where", ["first", "middle", "segment_boundary", "last"])
def test_memtest_injected_fault_latches_until_reset(P, where):
    max_bytes = GiB + 64 * MiB
    n_words = max_bytes // 4
    word = {"first": 0, "middle": 123457, "segment_boundary": GiB // 4, "last": n_words - 1}[where]
    with _open(P) as ctx:
        (r,) = ctx.memtest(0, max_bytes=max_bytes, fault_word=word, fault_mask=0x10)
        assert r.bytes_tested == max_bytes, r
        want = mt.march([16], 0, [(min(word, 15), 0x10)])                     # the counts do not depend on the size
        assert r.mismatches == [w[1] for w in want] == [0, 1, 1, 1]
        assert r.first_bad_word == word and not r.healthy and r.err == 0
        (p,) = ctx.probe_health(min_gbs=1e-3)
        assert p.flags & P._native.RES_MEMTEST and not p.healthy and p.mismatches == 0
        wire, st = ctx.list_and_watch("gpu", P._native.LW_HEARTBEAT, min_gbs=1e-3)
        assert st.n_unhealthy == 1
        ctx.probe_reset(0)
        (p,) = ctx.probe_health(min_gbs=1e-3)
        assert p.healthy and not p.flags & P._native.RES_MEMTEST


def test_memtest_leaves_the_probe_ring_alone(P):
    nbytes = 64 * MiB
    n_words = nbytes // 4
    with _open(P, nbytes) as ctx:
        (p0,) = ctx.probe_health(min_gbs=1e-3)
        seed = oprobe.next_seed(p0.seed)
        src = ctx.probe_peek(0, 0, n_words)
        assert np.array_equal(src, oprobe.pattern(n_words, seed))
        (r,) = ctx.memtest(0, max_bytes=512 * MiB)
        assert r.healthy
        assert np.array_equal(ctx.probe_peek(0, 0, n_words), src)
        (p,) = ctx.probe_health(min_gbs=1e-3)
        cs, bad, first, dst = oprobe.probe_pass(src, seed, oprobe.next_seed(seed))
        assert (p.seed, p.checksum, p.mismatches, p.first_bad_word) == (seed, cs, bad, first) and p.healthy
        assert np.array_equal(ctx.probe_peek(0, 0, n_words), dst)


def test_memtest_out_of_range_fault_is_not_injected(P):
    with _open(P) as ctx:
        (r,) = ctx.memtest(0, max_bytes=64 * MiB, fault_word=64 * MiB // 4, fault_mask=1)
        assert r.err == P._native.E_INVAL and r.mismatches == [0, 0, 0, 0] and r.healthy


def test_memtest_skips_a_busy_gpu(P):
    import torch
    helper = subprocess.Popen([sys.executable, "-c",
                               "import torch,time; torch.zeros(1, device='cuda:0'); print('ready', flush=True); time.sleep(60)"],
                              stdout=subprocess.PIPE, text=True)
    try:
        assert helper.stdout.readline().strip() == "ready"
        try:
            import pynvml
            pynvml.nvmlInit()
            seen = len(pynvml.nvmlDeviceGetComputeRunningProcesses(pynvml.nvmlDeviceGetHandleByIndex(0)))
        except Exception as e:       # noqa: BLE001
            pytest.skip("NVML process accounting unavailable: %s" % e)
        if seen < 1:
            pytest.skip("NVML does not list foreign compute processes in this container")
        with _open(P) as ctx:
            free0, _ = torch.cuda.mem_get_info(0)
            (r,) = ctx.memtest(0, max_bytes=256 * MiB)
            assert r.flags & P._native.MT_SKIPPED_BUSY and r.bytes_tested == 0 and r.n_segments == 0, r
            assert abs(torch.cuda.mem_get_info(0)[0] - free0) < 2 * MiB
            (p,) = ctx.probe_health(min_gbs=1e-3)
            assert not p.flags & P._native.RES_MEMTEST
            (r,) = ctx.memtest(0, max_bytes=256 * MiB, even_if_busy=True)
            assert not r.flags & P._native.MT_SKIPPED_BUSY and r.bytes_tested == 256 * MiB and r.healthy
    finally:
        if helper.poll() is None:
            helper.kill()
        helper.wait()


def _daemon_memtest_lines(short_dir, level):
    exe = os.path.join(ROOT, "k8s-device-plugin_b200", "b200dp_plugind")
    proc = subprocess.Popen([exe, "-backend=cuda:devices=0,bytes=67108864,calib=1", "-plugin_dir", short_dir,
                             "-start_retry_wait=0.05", "-memtest_at_start=%d" % level, "-memtest_max_bytes=268435456"],
                            stderr=subprocess.PIPE, text=True)
    lines = []
    try:
        t0 = time.time()
        while time.time() - t0 < 120:
            line = proc.stderr.readline()
            if not line:
                break
            lines.append(line)
            if "Failed to start plugin" in line:
                break
    finally:
        proc.send_signal(signal.SIGINT)
        rest = proc.communicate(timeout=30)[1]
    log = "".join(lines) + rest
    assert proc.returncode == 0, log[-3000:]
    assert log.index("memtest ") < log.index("Failed to start plugin"), log[-3000:]    # before the first registration
    return [ln for ln in log.splitlines() if ln.startswith("memtest ")], log


def test_daemon_memtest_at_start_logs_a_clean_result(short_dir):
    """-memtest_at_start=1 tests the GPU after open and before registering.  This test's own process holds a CUDA
    context, which NVML may list as another user of the GPU: then =1 skips it (nothing tested) and =2 tests it."""
    mem, log = _daemon_memtest_lines(short_dir, 1)
    assert len(mem) == 1, log[-3000:]
    if "flags 0x1," in mem[0]:
        assert ": Healthy, 0 bytes in 0 segment(s)" in mem[0]
        mem, log = _daemon_memtest_lines(short_dir, 2)
        assert len(mem) == 1, log[-3000:]
    assert ": Healthy, 268435456 bytes in 1 segment(s), flags 0x0" in mem[0].replace("flags 0x10", "flags 0x0"), log[-3000:]
