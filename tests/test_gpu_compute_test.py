"""The on-demand tensor-core self-test on a real H100.

- The kernel of tc_selftest.cuh, launched directly (tests/native/libcompute_test_kernels_test.so):
  - the DUMP instantiation's raw accumulators equal tests/compute_test_oracle.py bit for bit, for every format and
    tile at two seeds.  This is the measurement behind the exactness bounds in compute_test_math.hpp (BF16 partial
    sums up to 256 * 255^2 < 2^24, FP8 up to 7200 < 2^13);
  - a clean run covers every SM id and every CTA compares exactly what its rounds hold;
  - an injected fault on the first, a middle and the last SM id, on bit 0 and bit 31, is counted once by every CTA that
    ran on that SM and by no other.
- b2dp_compute_test through the ABI: Healthy on an idle card, memory handed back, the probe ring untouched, the fault
  hook attributed to its SM and latched until probe_reset, the busy skip, and the daemon's -compute_test_at_start.

Every run is short: 10-100 ms per format."""
import ctypes as C
import os
import signal
import subprocess
import sys
import time

import numpy as np
import pytest

import compute_test_oracle as ct
from oracle import probe as oprobe

pytestmark = pytest.mark.gpu

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(HERE)
LIB_PATH = os.path.join(HERE, "native", "libcompute_test_kernels_test.so")
MiB = 1 << 20
MS = 1000000


class CtRecord(C.Structure):
    _fields_ = [("smid", C.c_uint32), ("nsmid", C.c_uint32), ("rounds", C.c_uint64), ("comparisons", C.c_uint64),
                ("mismatches", C.c_uint64), ("first_bad_tile", C.c_int32), ("first_bad_rep", C.c_int32),
                ("seq", C.c_uint64)]


class Harness:
    def __init__(self, device=0):
        L = C.CDLL(LIB_PATH)
        L.ck_open.restype = C.c_void_p
        L.ck_open.argtypes = [C.c_int, C.c_char_p, C.c_int]
        L.ck_close.argtypes = [C.c_void_p]
        L.ck_error.restype = C.c_char_p
        L.ck_error.argtypes = [C.c_void_p]
        L.ck_sms.argtypes = [C.c_void_p]
        L.ck_occupancy.argtypes = [C.c_void_p, C.c_int, C.POINTER(C.c_int)]
        L.ck_dump.argtypes = [C.c_void_p, C.c_int, C.c_uint32, C.POINTER(C.c_uint32), C.POINTER(CtRecord)]
        L.ck_run.argtypes = [C.c_void_p, C.c_int, C.c_uint32, C.c_uint64, C.c_int, C.c_uint32, C.POINTER(CtRecord), C.c_int,
                             C.POINTER(C.c_int), C.POINTER(C.c_float)]
        assert L.ck_record_bytes() == C.sizeof(CtRecord)
        assert (L.ck_tiles(), L.ck_reps()) == (ct.TILES, ct.REPS)
        self.L = L
        err = C.create_string_buffer(512)
        self.h = L.ck_open(device, err, len(err))
        if not self.h:
            raise RuntimeError("ck_open: " + err.value.decode())
        self.sms = L.ck_sms(self.h)

    def close(self):
        if self.h:
            self.L.ck_close(self.h)
            self.h = None

    def _check(self, rc, what):
        if rc == 1:
            raise RuntimeError("%s: %s" % (what, self.L.ck_error(self.h).decode()))
        assert rc == 0, "%s refused: code %d" % (what, rc)

    def occupancy(self, fmt):
        n = C.c_int()
        self._check(self.L.ck_occupancy(self.h, fmt, C.byref(n)), "ck_occupancy")
        return n.value

    def dump(self, fmt, seed):
        out = np.zeros(ct.TILES * ct.THREADS * ct.ACC, dtype=np.uint32)
        rec = CtRecord()
        self._check(self.L.ck_dump(self.h, fmt, seed, out.ctypes.data_as(C.POINTER(C.c_uint32)), C.byref(rec)), "ck_dump")
        return out.reshape(ct.TILES, ct.THREADS, ct.ACC), rec

    def run(self, fmt, seed, duration_ms, fault_sm=-1, fault_mask=0):
        cap = self.sms * 32
        recs = (CtRecord * cap)()
        n, ms = C.c_int(), C.c_float()
        self._check(self.L.ck_run(self.h, fmt, seed, int(duration_ms * MS), fault_sm, fault_mask, recs, cap, C.byref(n),
                                  C.byref(ms)), "ck_run")
        return list(recs[:n.value]), ms.value


@pytest.fixture(scope="module")
def H():
    if not os.path.exists(LIB_PATH):
        pytest.skip("run __graft_entry__.build() first")
    h = Harness(0)
    yield h
    h.close()


def _gpu_busy():
    """True if NVML lists a compute process on GPU 0 besides this one, which holds a context itself (the rule
    b2dp_compute_test applies; NVML's pids are the host's, not this container's).  None if NVML cannot tell."""
    try:
        import pynvml
        pynvml.nvmlInit()
        return len(pynvml.nvmlDeviceGetComputeRunningProcesses(pynvml.nvmlDeviceGetHandleByIndex(0))) > 1
    except Exception:       # noqa: BLE001
        return None


# ---- the kernel, directly ---------------------------------------------------------------------------------------------
@pytest.mark.parametrize("seed", [0x0, 0xC0FFEE17])
@pytest.mark.parametrize("fmt", ct.FORMATS, ids=[ct.NAMES[f] for f in ct.FORMATS])
def test_dump_matches_the_exact_product_bit_for_bit(H, fmt, seed):
    got, rec = H.dump(fmt, seed)
    bad = []
    for t in range(ct.TILES):
        d = ct.tile(seed, fmt, t)[4]
        want = ct.fragments(d)
        if not np.array_equal(got[t], want):
            idx = np.argwhere(got[t] != want)
            th, j = idx[0]
            bad.append("tile %d: %d of %d words differ; first thread %d reg %d got 0x%08x want 0x%08x"
                       % (t, len(idx), want.size, th, j, got[t][th, j], want[th, j]))
    assert not bad, "\n".join(bad)
    # and the kernel's own comparison agreed: one round, every repetition compared, none mismatched
    assert (rec.seq, rec.rounds, rec.comparisons, rec.mismatches) == (1, 1, ct.TILES * ct.REPS, 0), \
        (rec.seq, rec.rounds, rec.comparisons, rec.mismatches)
    assert (rec.first_bad_tile, rec.first_bad_rep) == (-1, -1)


def _check_clean(H, recs):
    for r in recs:
        assert r.seq == 7 and r.rounds >= 1 and r.comparisons == r.rounds * ct.TILES * ct.REPS, \
            (r.smid, r.seq, r.rounds, r.comparisons)
        assert r.mismatches == 0 and (r.first_bad_tile, r.first_bad_rep) == (-1, -1)
        assert r.smid < r.nsmid <= 256


@pytest.fixture(scope="module")
def sm_ids(H):
    """The %smid values a clean BF16 run covered (sorted)."""
    recs, _ = H.run(ct.BF16, 0x5EED, 20)
    _check_clean(H, recs)
    return sorted({r.smid for r in recs})


@pytest.mark.parametrize("fmt", ct.FORMATS, ids=[ct.NAMES[f] for f in ct.FORMATS])
def test_clean_run_covers_every_sm(H, fmt):
    duration = 100
    recs, ms = H.run(fmt, 0x1234567 + fmt, duration)
    assert len(recs) == H.sms * H.occupancy(fmt)
    _check_clean(H, recs)
    assert ms >= duration * 0.9
    per_sm = np.bincount([r.smid for r in recs])
    ops = 2 * ct.M * ct.N * ct.K[fmt] * sum(r.comparisons for r in recs)
    print("%s: %d CTAs (%d resident per SM; per SM id min %d max %d), %d SM ids, %.1f ms, %.0f T%s/s"
          % (ct.NAMES[fmt], len(recs), H.occupancy(fmt), per_sm[per_sm > 0].min(), per_sm.max(), len(set(r.smid for r in recs)),
             ms, ops / ms * 1e-9, "OP" if fmt == ct.INT8 else "FLOP"))
    if _gpu_busy():
        pytest.skip("another process uses the GPU: coverage is not asserted (the rest was)")
    assert len({r.smid for r in recs}) == H.sms, (len({r.smid for r in recs}), H.sms)


@pytest.mark.parametrize("mask", [0x1, 0x80000000], ids=["bit0", "bit31"])
@pytest.mark.parametrize("where", ["first", "middle", "last"])
def test_injected_fault_is_counted_by_every_cta_on_its_sm(H, sm_ids, where, mask):
    s = {"first": sm_ids[0], "middle": sm_ids[len(sm_ids) // 2], "last": sm_ids[-1]}[where]
    for fmt in ct.FORMATS:
        recs, _ = H.run(fmt, 0xFA017 + fmt, 10, fault_sm=s, fault_mask=mask)
        on_s = [r for r in recs if r.smid == s]
        assert on_s, "no CTA ran on SM %d" % s
        for r in recs:
            assert r.seq == 7 and r.comparisons == r.rounds * ct.TILES * ct.REPS
            if r.smid == s:
                assert (r.mismatches, r.first_bad_tile, r.first_bad_rep) == (1, 0, 0), (ct.NAMES[fmt], r.smid, r.mismatches)
            else:
                assert r.mismatches == 0, (ct.NAMES[fmt], r.smid, r.mismatches)


# ---- through the ABI --------------------------------------------------------------------------------------------------
def _open(pkg, nbytes=64 * MiB):
    return pkg.Context("cuda:devices=0,bytes=%d,calib=1" % nbytes)


def test_compute_test_clean_memory_back_and_ring_untouched(pkg):
    import torch
    torch.cuda.init()
    N = pkg._native
    nbytes = 64 * MiB
    n_words = nbytes // 4
    with _open(pkg, nbytes) as ctx:
        ctx.compute_test(0, duration_ms=10)                   # first launch loads the kernels: not counted below
        (p0,) = ctx.probe_health(min_gbs=1e-3)
        seed = oprobe.next_seed(p0.seed)
        src = ctx.probe_peek(0, 0, n_words)
        free0, _ = torch.cuda.mem_get_info(0)
        (r,) = ctx.compute_test(0, duration_ms=100)
        free1, _ = torch.cuda.mem_get_info(0)
        assert r.healthy and r.err == 0, r
        assert r.mismatches == [0, 0, 0] and r.bad_sm_mask == [0, 0, 0, 0], r
        assert (r.first_bad_sm, r.first_bad_format, r.first_bad_tile) == (-1, -1, -1)
        assert r.sm_count == torch.cuda.get_device_properties(0).multi_processor_count
        assert r.nsmid >= r.sm_count and all(ms >= 90 for ms in r.ms) and all(t > 0 for t in r.tflops), r
        if not _gpu_busy():
            assert r.sms_covered == r.sm_count and not r.flags & N.CT_PARTIAL_COVERAGE, r
        assert abs(free1 - free0) < 2 * MiB, (free0, free1)  # every allocation was released before the call returned
        assert np.array_equal(ctx.probe_peek(0, 0, n_words), src)
        (p,) = ctx.probe_health(min_gbs=1e-3)
        cs, bad, first, _ = oprobe.probe_pass(src, seed, oprobe.next_seed(seed))
        assert (p.seed, p.checksum, p.mismatches) == (seed, cs, bad) and p.healthy
        assert not p.flags & N.RES_COMPUTE
    print("compute test 100 ms/format: SMs %d/%d, ms %s, TFLOP/s bf16 %.0f fp8 %.0f, TOPS int8 %.0f"
          % (r.sms_covered, r.sm_count, ["%.1f" % x for x in r.ms], *r.tflops))


@pytest.mark.parametrize("where,mask", [("first", 0x1), ("middle", 0x80000000), ("last", 0x1)])
def test_compute_test_fault_is_attributed_and_latched_until_reset(pkg, H, sm_ids, where, mask):
    N = pkg._native
    s = {"first": sm_ids[0], "middle": sm_ids[len(sm_ids) // 2], "last": sm_ids[-1]}[where]
    with _open(pkg) as ctx:
        (r,) = ctx.compute_test(0, duration_ms=10, fault_sm=s, fault_mask=mask)
        assert not r.healthy and r.err == 0, r
        assert r.bad_sms() == [s], r.bad_sms()
        assert (r.first_bad_sm, r.first_bad_format, r.first_bad_tile) == (s, ct.BF16, 0), r
        for f in ct.FORMATS:          # one mismatch per CTA that ran on s: between 1 and the resident CTAs per SM
            assert 1 <= r.mismatches[f] <= H.occupancy(f), (f, r.mismatches)
        (p,) = ctx.probe_health(min_gbs=1e-3)
        assert p.flags & N.RES_COMPUTE and not p.healthy and p.mismatches == 0
        _, st = ctx.list_and_watch("gpu", N.LW_HEARTBEAT, min_gbs=1e-3)
        assert st.n_unhealthy == 1
        ctx.probe_reset(0)
        (p,) = ctx.probe_health(min_gbs=1e-3)
        assert p.healthy and not p.flags & N.RES_COMPUTE


def test_compute_test_skips_a_busy_gpu(pkg):
    N = pkg._native
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
        with _open(pkg) as ctx:
            (r,) = ctx.compute_test(0, duration_ms=10, fault_sm=0, fault_mask=1)
            assert r.flags & N.CT_SKIPPED_BUSY and r.mismatches == [0, 0, 0] and r.ms == [0, 0, 0], r
            (p,) = ctx.probe_health(min_gbs=1e-3)
            assert not p.flags & N.RES_COMPUTE                 # nothing ran, nothing latched
            (r,) = ctx.compute_test(0, duration_ms=10, even_if_busy=True)
            assert not r.flags & N.CT_SKIPPED_BUSY and r.healthy and r.err == 0, r
    finally:
        if helper.poll() is None:
            helper.kill()
        helper.wait()


def _daemon_lines(short_dir, level):
    exe = os.path.join(ROOT, "k8s-device-plugin_b200", "b200dp_plugind")
    proc = subprocess.Popen([exe, "-backend=cuda:devices=0,bytes=67108864,calib=1", "-plugin_dir", short_dir,
                             "-start_retry_wait=0.05", "-compute_test_at_start=%d" % level, "-compute_test_ms=50"],
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
    assert log.index("compute test ") < log.index("Failed to start plugin"), log[-3000:]  # before the first registration
    return [ln for ln in log.splitlines() if ln.startswith("compute test ")], log


def test_daemon_compute_test_at_start_logs_a_clean_result(short_dir):
    """-compute_test_at_start=1 tests the GPU after open and before registering.  This test's own process may hold a
    CUDA context, which NVML may list as another user of the GPU: then =1 skips it and =2 tests it."""
    lines, log = _daemon_lines(short_dir, 1)
    assert len(lines) == 1, log[-3000:]
    if "flags 0x1," in lines[0]:
        lines, log = _daemon_lines(short_dir, 2)
        assert len(lines) == 1, log[-3000:]
    assert ": Healthy, flags 0x" in lines[0] and "mismatches 0/0/0, first bad SM -1" in lines[0], log[-3000:]
