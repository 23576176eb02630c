"""The on-demand host-link self-test on a real H100.

- The SM format's kernel (hostlink_selftest.cuh), launched directly through tests/native/libhostlink_kernels_test.so on
  mapped pinned host buffers, against tests/hostlink_oracle.py at ragged sizes: the destination buffer bit for bit, a
  guard region past it, the checksum against the host's closed form, the per-CTA records (every SM id, every vector
  once), and the fault hook at the first, a middle and the last word.
- b2dp_hostlink_test through the ABI: a clean run, the NVML link fields, the fault hook in every format, the latch and
  its reset, an out-of-range fault word, rejected sizes, device memory handed back, a second call, the busy skip, and
  the daemon's -hostlink_test_at_start.

No rate threshold is asserted: what a host's root complex carries is not a property of the GPU."""
import ctypes as C
import os
import signal
import subprocess
import sys
import time

import numpy as np
import pytest

import hostlink_oracle as hl
from oracle import probe as oprobe

pytestmark = pytest.mark.gpu

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(HERE)
LIB_PATH = os.path.join(HERE, "native", "libhostlink_kernels_test.so")
MiB, GiB = 1 << 20, 1 << 30
U64 = C.c_uint64
GUARD_WORDS = 1024
SENTINEL = 0xA5A5A5A5


class ProbeOut(C.Structure):
    _fields_ = [("checksum", U64), ("mismatches", U64), ("first_bad", U64), ("t_start_ns", U64), ("t_end_ns", U64),
                ("seq", U64)]


class HlRecord(C.Structure):
    _fields_ = [("seq", U64), ("vectors", U64), ("mismatches", U64), ("smid", C.c_uint32), ("nsmid", C.c_uint32)]


class Harness:
    def __init__(self, device=0):
        L = C.CDLL(LIB_PATH)
        L.hk_open.restype = C.c_void_p
        L.hk_open.argtypes = [C.c_int, C.c_char_p, C.c_int]
        L.hk_close.argtypes = [C.c_void_p]
        L.hk_error.restype = C.c_char_p
        L.hk_error.argtypes = [C.c_void_p]
        L.hk_sms.argtypes = [C.c_void_p]
        L.hk_grid.argtypes = [C.c_void_p]
        L.hk_alloc.argtypes = [C.c_void_p, U64, C.POINTER(C.c_void_p), C.POINTER(C.c_void_p)]
        L.hk_run.argtypes = [C.c_void_p, U64, C.c_uint32, C.c_uint32, U64, C.c_uint32, C.c_int, U64,
                             C.POINTER(ProbeOut), C.POINTER(HlRecord), C.c_int]
        self.L = L
        assert L.hk_record_bytes() == C.sizeof(HlRecord)
        err = C.create_string_buffer(512)
        self.h = L.hk_open(device, err, len(err))
        if not self.h:
            raise RuntimeError("hk_open: " + err.value.decode())
        self.sms = L.hk_sms(self.h)
        self.grid = L.hk_grid(self.h)
        self.seq = 0

    def close(self):
        if self.h:
            self.L.hk_close(self.h)
            self.h = None

    def _check(self, rc, what):
        if rc == 1:
            raise RuntimeError("%s: %s" % (what, self.L.hk_error(self.h).decode()))
        assert rc == 0, "%s refused: code %d" % (what, rc)

    def alloc(self, n_words):
        """Two mapped host buffers of n_words words, as numpy views."""
        src, dst = C.c_void_p(), C.c_void_p()
        self._check(self.L.hk_alloc(self.h, n_words * 4, C.byref(src), C.byref(dst)), "hk_alloc")
        view = lambda p: np.ctypeslib.as_array((C.c_uint32 * n_words).from_address(p.value))  # noqa: E731
        return view(src), view(dst)

    def run(self, n_vec, seed, nxt, fault_word=0, fault_mask=0, grid=0):
        self.seq += 1
        out = ProbeOut()
        g = grid or self.grid
        recs = (HlRecord * g)()
        rc = self.L.hk_run(self.h, n_vec, seed, seed ^ nxt, fault_word, fault_mask, grid, self.seq, C.byref(out),
                           recs, g)
        self._check(rc, "hk_run")
        return out, list(recs)


@pytest.fixture(scope="module")
def H():
    if not os.path.exists(LIB_PATH):
        pytest.skip("run __graft_entry__.build() first")
    h = Harness(0)
    yield h
    h.close()


def _pass(H, n_vec, seed, fault_word=0, fault_mask=0):
    """One SM-format pass over n_vec vectors with a guard region past them, checked against the oracle."""
    n_words = 4 * n_vec
    src, dst = H.alloc(n_words + GUARD_WORDS)
    src[:n_words] = oprobe.pattern(n_words, seed)
    src[n_words:] = SENTINEL
    dst[:] = SENTINEL
    nxt = hl.next_seed(seed)
    out, recs = H.run(n_vec, seed, nxt, fault_word, fault_mask)
    cs, bad, first, want = hl.sm_pass(np.array(src[:n_words]), seed, nxt, fault_word, fault_mask)
    assert out.seq == H.seq
    assert (out.checksum, out.mismatches, out.first_bad) == (cs, bad, first), (n_vec, fault_word)
    if not fault_mask:
        assert out.checksum == oprobe.expected_checksum(n_words, seed)
    assert np.array_equal(dst[:n_words], want), np.nonzero(dst[:n_words] != want)[0][:8]
    assert np.all(dst[n_words:] == SENTINEL), "the kernel wrote past n_vec"
    assert np.all(src[n_words:] == SENTINEL)
    assert all(r.seq == H.seq for r in recs), "a CTA record did not arrive"
    assert sum(r.vectors for r in recs) == n_vec
    assert sum(r.mismatches for r in recs) == bad
    assert len({r.smid for r in recs}) == H.sms, sorted({r.smid for r in recs})
    return out, recs, dst


@pytest.mark.parametrize("n_vec", [1, 31, (1 << 20) + 3, (64 * MiB) // 16], ids=["1", "31", "2^20+3", "default"])
def test_sm_kernel_matches_oracle(H, n_vec):
    _pass(H, n_vec, 0x5EED0000 ^ n_vec)


@pytest.mark.parametrize("where", ["first", "middle", "last"])
def test_sm_kernel_fault_counted_once(H, where):
    n_vec = (1 << 20) + 3
    word = {"first": 0, "middle": 2 * n_vec + 1, "last": 4 * n_vec - 1}[where]
    out, recs, dst = _pass(H, n_vec, 0xFA017000, word, 0x10)
    assert (out.mismatches, out.first_bad) == (1, word)
    assert sum(1 for r in recs if r.mismatches) == 1
    assert hl.check(np.array(dst[:4 * n_vec]), hl.next_seed(0xFA017000)) == (1, word)


# ---- through the ABI --------------------------------------------------------------------------------------------------
@pytest.fixture(scope="module")
def P(pkg):
    return pkg


def _open(P):
    return P.Context("cuda:devices=0,bytes=%d,calib=1" % (64 * MiB))


def _check_link(P, r):
    if r.flags & P._native.HL_NO_NVML:
        return
    assert 1 <= r.link_gen <= r.max_link_gen, r
    assert 1 <= r.link_width <= r.max_link_width, r
    assert abs(r.link_gbs - hl.link_gbs(r.link_gen, r.link_width)) < 1e-3


def test_hostlink_clean_run_memory_back_and_second_call(P):
    import torch
    torch.cuda.init()
    with _open(P) as ctx:
        ctx.hostlink_test(0, bytes=MiB, duration_ms=20)              # first launch loads the kernels
        free0, _ = torch.cuda.mem_get_info(0)
        (r,) = ctx.hostlink_test(0, duration_ms=300)
        free1, _ = torch.cuda.mem_get_info(0)
        assert r.healthy and r.err == 0, r
        assert r.mismatches == [0, 0, 0] and r.first_bad_word == [hl.NO_BAD] * 3
        assert all(k >= 1 for k in r.rounds) and all(g > 0 for g in r.gbs) and all(m > 0 for m in r.ms), r
        for f in (hl.H2D, hl.D2H):
            assert abs(r.gbs[f] - 64 * MiB * r.rounds[f] / r.ms[f] * 1e-6) < 1e-3 * r.gbs[f]
        assert abs(r.gbs[hl.SM] - 2 * 64 * MiB * r.rounds[hl.SM] / r.ms[hl.SM] * 1e-6) < 1e-3 * r.gbs[hl.SM]
        assert r.sms_covered == r.sm_count and r.bad_sm_mask == [0, 0, 0, 0]
        assert not r.flags & P._native.HL_SKIPPED_BUSY
        assert (r.host_numa_node >= 0) != bool(r.flags & P._native.HL_NUMA_UNBOUND)
        _check_link(P, r)
        assert abs(free1 - free0) < 2 * MiB, (free0, free1)          # every buffer was freed before the call returned
        (r2,) = ctx.hostlink_test(0, bytes=4 * MiB, duration_ms=50)
        assert r2.healthy and r2.err == 0, r2
        (p,) = ctx.probe_health(min_gbs=1e-3)
        assert p.healthy and not p.flags & P._native.RES_HOSTLINK
    print("hostlink 64 MiB: h2d %.2f d2h %.2f sm %.2f GB/s, rounds %s, PCIe gen %d/%d x%d/%d (%.1f GB/s), "
          "replays %d, numa %d, flags 0x%x" % (r.gbs[0], r.gbs[1], r.gbs[2], r.rounds, r.link_gen, r.max_link_gen,
                                              r.link_width, r.max_link_width, r.link_gbs, r.replays,
                                              r.host_numa_node, r.flags))


@pytest.mark.parametrize("where", ["first", "middle", "last"])
def test_hostlink_fault_caught_in_every_format_and_latched_until_reset(P, where):
    nbytes = 4 * MiB
    n_words = nbytes // 4
    word = {"first": 0, "middle": 123457, "last": n_words - 1}[where]
    with _open(P) as ctx:
        (r,) = ctx.hostlink_test(0, bytes=nbytes, duration_ms=50, fault_word=word, fault_mask=0x10)
        assert not r.healthy and r.err == 0, r
        # H2D: the kernel sees the word on the device, the host sees it again after the re-key; D2H: the host only;
        # SM: the kernel as it reads it, then the host
        assert r.mismatches == [2, 1, 2], r
        assert r.first_bad_word == [word] * 3
        assert r.bad_sm_mask != [0, 0, 0, 0]
        (p,) = ctx.probe_health(min_gbs=1e-3)
        assert p.flags & P._native.RES_HOSTLINK and not p.healthy and p.mismatches == 0
        wire, st = ctx.list_and_watch("gpu", P._native.LW_HEARTBEAT, min_gbs=1e-3)
        assert st.n_unhealthy == 1
        ctx.probe_reset(0)
        (p,) = ctx.probe_health(min_gbs=1e-3)
        assert p.healthy and not p.flags & P._native.RES_HOSTLINK


def test_hostlink_out_of_range_fault_is_not_injected(P):
    with _open(P) as ctx:
        (r,) = ctx.hostlink_test(0, bytes=MiB, duration_ms=30, fault_word=MiB // 4, fault_mask=1)
        assert r.err == P._native.E_INVAL and r.mismatches == [0, 0, 0] and r.healthy, r


@pytest.mark.parametrize("nbytes", [17, 8, GiB + 16, 2 * GiB])
def test_hostlink_rejects_bad_sizes(P, nbytes):
    with _open(P) as ctx:
        with pytest.raises(P._native.B2dpError) as ei:
            ctx.hostlink_test(0, bytes=nbytes, duration_ms=10)
        assert ei.value.code == P._native.E_INVAL


def test_hostlink_skips_a_busy_gpu(P):
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
            (r,) = ctx.hostlink_test(0, bytes=MiB, duration_ms=20)
            assert r.flags & P._native.HL_SKIPPED_BUSY and r.rounds == [0, 0, 0], r
            (p,) = ctx.probe_health(min_gbs=1e-3)
            assert not p.flags & P._native.RES_HOSTLINK
            (r,) = ctx.hostlink_test(0, bytes=MiB, duration_ms=20, even_if_busy=True)
            assert not r.flags & P._native.HL_SKIPPED_BUSY and r.healthy, r
    finally:
        if helper.poll() is None:
            helper.kill()
        helper.wait()


def _daemon_hostlink_lines(short_dir, level):
    exe = os.path.join(ROOT, "k8s-device-plugin_b200", "b200dp_plugind")
    proc = subprocess.Popen([exe, "-backend=cuda:devices=0,bytes=67108864,calib=1", "-plugin_dir", short_dir,
                             "-start_retry_wait=0.05", "-hostlink_test_at_start=%d" % level, "-compute_test_ms=100"],
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
    assert log.index("host-link test ") < log.index("Failed to start plugin"), log[-3000:]
    return [ln for ln in log.splitlines() if ln.startswith("host-link test ")], log


def test_daemon_hostlink_test_at_start(short_dir):
    """-hostlink_test_at_start=1 tests the GPU after open and before registering.  This test's own process may hold a
    CUDA context, which NVML may list as another user of the GPU: then =1 skips it and =2 tests it."""
    hl_lines, log = _daemon_hostlink_lines(short_dir, 1)
    assert len(hl_lines) == 1, log[-3000:]
    if int(hl_lines[0].split("flags ")[1].split(",")[0], 16) & 0x1:
        hl_lines, log = _daemon_hostlink_lines(short_dir, 2)
        assert len(hl_lines) == 1, log[-3000:]
    assert ": Healthy, " in hl_lines[0] and "mismatches 0/0/0" in hl_lines[0], log[-3000:]
