"""GPU tests of the on-demand L2 self-test (b2dp_l2_test, csrc/l2_selftest.cuh).

- The kernel of l2_selftest.cuh, launched cooperatively through tests/native/libl2_test_kernels_test.so:
  - the DUMP of every format equals tests/l2_test_oracle.py bit for bit: every CTA's folds and error counts and the
    window image after the march (WORD, BYTE), the hot block and the combined folds the checker saw (ATOM);
  - every CTA is co-resident and all run the same rounds, with complete, clean records;
  - the fault hook's flip is counted in exactly the first comparison, by exactly the CTA that reads the word: the
    next owner for WORD and BYTE, the checker of comparison 0 (CTA 0) for ATOM.
- b2dp_l2_test through the ABI: Healthy on an idle card with every SM id covered, the fault hook attributed and
  latched until probe_reset, the busy skip, free memory unchanged, and the daemon's -l2_test_at_start.
"""
import ctypes as C
import os
import signal
import subprocess
import sys
import time

import numpy as np
import pytest

import l2_test_oracle as lo

pytestmark = pytest.mark.gpu

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(HERE)
LIB_PATH = os.path.join(HERE, "native", "libl2_test_kernels_test.so")
MiB = 1 << 20
MS = 1000000
FORMATS = (lo.WORD, lo.BYTE, lo.ATOM)
FMT_IDS = ["word", "byte", "atom"]


class CtRecord(C.Structure):
    _fields_ = [("smid", C.c_uint32), ("nsmid", C.c_uint32), ("rounds", C.c_uint64), ("comparisons", C.c_uint64),
                ("mismatches", C.c_uint64), ("first_bad_tile", C.c_int32), ("first_bad_rep", C.c_int32),
                ("seq", C.c_uint64)]


_P = C.POINTER


class Harness:
    def __init__(self, device=0):
        L = C.CDLL(LIB_PATH)
        L.lk_open.restype = C.c_void_p
        L.lk_open.argtypes = [C.c_int, C.c_char_p, C.c_int]
        L.lk_close.argtypes = [C.c_void_p]
        L.lk_error.restype = C.c_char_p
        L.lk_error.argtypes = [C.c_void_p]
        L.lk_sms.argtypes = [C.c_void_p]
        L.lk_l2_bytes.argtypes = [C.c_void_p]
        L.lk_occupancy.argtypes = [C.c_void_p, C.c_int, C.c_int, _P(C.c_int)]
        L.lk_dump_words.restype = C.c_uint64
        L.lk_dump_words.argtypes = [C.c_int, C.c_int, C.c_uint]
        L.lk_run.argtypes = [C.c_void_p, C.c_int, C.c_int, C.c_uint32, C.c_uint, C.c_uint64, C.c_int, C.c_uint32,
                             _P(CtRecord), C.c_int, _P(C.c_int), _P(C.c_float), _P(C.c_uint), _P(C.c_uint32)]
        assert L.lk_record_bytes() == C.sizeof(CtRecord)
        self.L = L
        err = C.create_string_buffer(512)
        self.h = L.lk_open(device, err, len(err))
        if not self.h:
            raise RuntimeError("lk_open: " + err.value.decode())
        self.sms = L.lk_sms(self.h)
        self.l2 = L.lk_l2_bytes(self.h)

    def close(self):
        if self.h:
            self.L.lk_close(self.h)
            self.h = None

    def occupancy(self, fmt, dump=False):
        n = C.c_int()
        rc = self.L.lk_occupancy(self.h, fmt, int(dump), C.byref(n))
        assert rc == 0, self.L.lk_error(self.h)
        return n.value

    def run(self, fmt, seed, duration_ms, K=0, fault_sm=-1, fault_mask=0, dump=False):
        grid = self.sms * self.occupancy(fmt, dump)
        recs = (CtRecord * grid)()
        n, ms, k = C.c_int(), C.c_float(), C.c_uint()
        out = None
        if dump:
            assert K, "a DUMP run takes an explicit span"
            out = np.zeros(self.L.lk_dump_words(fmt, grid, K), dtype=np.uint32)
        rc = self.L.lk_run(self.h, fmt, int(dump), seed, K, int(duration_ms * MS), fault_sm, fault_mask, recs, grid,
                           C.byref(n), C.byref(ms), C.byref(k), out.ctypes.data_as(_P(C.c_uint32)) if dump else None)
        if rc == 1:
            raise RuntimeError(self.L.lk_error(self.h).decode())
        assert rc == 0, rc
        return list(recs[:n.value]), ms.value, k.value, out


@pytest.fixture(scope="module")
def H():
    if not os.path.exists(LIB_PATH):
        pytest.skip("run __graft_entry__.build() first")
    h = Harness(0)
    yield h
    h.close()


def _gpu_busy():
    try:
        import pynvml
        pynvml.nvmlInit()
        return len(pynvml.nvmlDeviceGetComputeRunningProcesses(pynvml.nvmlDeviceGetHandleByIndex(0))) > 1
    except Exception:       # noqa: BLE001
        return None


def _check_clean(recs, seq=7):
    rounds = {r.rounds for r in recs}
    assert len(rounds) == 1, "CTAs ran different rounds: %s" % sorted(rounds)
    for r in recs:
        assert r.seq == seq and r.rounds >= 1 and r.comparisons == r.rounds * lo.TILES * lo.REPS, \
            (r.smid, r.seq, r.rounds, r.comparisons)
        assert r.mismatches == 0 and (r.first_bad_tile, r.first_bad_rep) == (-1, -1), \
            (r.smid, r.mismatches, r.first_bad_tile, r.first_bad_rep)


# ---- the kernel, directly ---------------------------------------------------------------------------------------------
@pytest.mark.parametrize("fmt", FORMATS, ids=FMT_IDS)
def test_dump_matches_the_oracle_bit_for_bit(H, fmt):
    seed, K = 0xC0FFEE17, 2
    recs, _, k, out = H.run(fmt, seed, 0, K=K, dump=True)
    G = len(recs)
    _check_clean(recs)
    assert all(r.rounds == 1 for r in recs)
    if fmt == lo.ATOM:
        d = out.reshape(lo.TILES, lo.ATOM_HOT_WORDS + 4 * lo.ATOM_RET)
        for t in range(lo.TILES):
            hot, folds = lo.atom_expected(seed, t, G)
            exch = np.array([lo.word_slot(i)[0] == lo.EXCH for i in range(lo.ATOM_HOT_WORDS)])
            got_hot = d[t, :lo.ATOM_HOT_WORDS]
            assert np.array_equal(got_hot[~exch], hot[~exch]), \
                (t, np.argwhere(got_hot != hot)[:5].ravel().tolist())
            _, X = lo.finals(seed, t)
            assert set(got_hot[exch].tolist()) <= set(X[lo.EXCH]) | {lo.init(seed, t, lo.EXCH)}, t
            got = d[t, lo.ATOM_HOT_WORDS:]
            assert np.array_equal(got[:2 * lo.ATOM_RET], got[2 * lo.ATOM_RET:]), (t, got)
            assert np.array_equal(got[2 * lo.ATOM_RET:], folds), (t, got, folds)
        return
    span = K * G * lo.BLOCK_WORDS
    folds = out[:lo.TILES * G * 2 * lo.THREADS].reshape(lo.TILES, G, 2, lo.THREADS)
    images = out[lo.TILES * G * 2 * lo.THREADS:].reshape(lo.TILES, span)
    for t in range(lo.TILES):
        table, checks = lo.tile(seed, fmt, t)
        assert (folds[t, :, 1, :] == 0).all(), t
        assert np.array_equal(folds[t, :, 0, :], np.tile((checks * np.uint32(K)).astype(np.uint32), (G, 1))), t
        assert np.array_equal(images[t], lo.window(table, span)), t


@pytest.mark.parametrize("fmt", FORMATS, ids=FMT_IDS)
def test_clean_run_is_co_resident_with_equal_rounds(H, fmt):
    duration = 100
    recs, ms, K, _ = H.run(fmt, 0x1234567 + fmt, duration)
    assert len(recs) == H.sms * H.occupancy(fmt)
    _check_clean(recs)
    assert ms >= duration * 0.9
    print("%s: %d CTAs, K %d (span %.2f MiB of a %d KiB L2), %d rounds, %.1f ms"
          % (FMT_IDS[fmt], len(recs), K, K * len(recs) * 2048 / MiB, H.l2 >> 10, recs[0].rounds, ms))
    if not _gpu_busy():
        assert len({r.smid for r in recs}) == H.sms
    if fmt != lo.ATOM:
        # the slice CTA c writes in element e is read by CTA c - 1 in element e + 1: every handoff crosses SMs
        G = len(recs)
        same = [c for c in range(G) if recs[c].smid == recs[(c - 1) % G].smid]
        assert not same, "%d of %d handoffs stay on one SM, first CTA %d" % (len(same), G, same[0])


@pytest.mark.parametrize("fmt", FORMATS, ids=FMT_IDS)
def test_fault_hook_is_counted_by_the_cta_that_reads_the_word(H, fmt):
    recs0, _, _, _ = H.run(lo.WORD, 0x5EED, 1)
    sm = recs0[len(recs0) // 2].smid
    recs, _, _, _ = H.run(fmt, 0xF00D, 5, fault_sm=sm, fault_mask=0x80000001)
    G = len(recs)
    bad = [c for c, r in enumerate(recs) if r.mismatches]
    assert len(bad) == 1, [(c, recs[c].mismatches) for c in bad]
    r = recs[bad[0]]
    assert (r.mismatches, r.first_bad_tile, r.first_bad_rep) == (1, 0, 0), (r.mismatches, r.first_bad_tile)
    if fmt == lo.ATOM:
        assert bad == [0]                                   # the checker of comparison 0
    else:
        assert recs[(bad[0] + 1) % G].smid == sm             # the previous owner ran on the faulted SM
    assert all(x.rounds == recs[0].rounds and x.comparisons == x.rounds * lo.TILES * lo.REPS for x in recs)


# ---- through the ABI --------------------------------------------------------------------------------------------------
def _open(pkg, nbytes=64 * MiB):
    return pkg.Context("cuda:devices=0,bytes=%d,calib=1" % nbytes)


def test_l2_test_clean_and_memory_back(pkg):
    import torch
    torch.cuda.init()
    N = pkg._native
    with _open(pkg) as ctx:
        ctx.l2_test(0, duration_ms=10)
        free0, _ = torch.cuda.mem_get_info(0)
        (r,) = ctx.l2_test(0, duration_ms=100)
        free1, _ = torch.cuda.mem_get_info(0)
        assert r.healthy and r.err == 0, r
        assert r.mismatches == [0, 0, 0] and r.bad_sm_mask == [0, 0, 0, 0], r
        assert r.sm_count == torch.cuda.get_device_properties(0).multi_processor_count
        assert all(ms >= 90 for ms in r.ms) and all(t > 0 for t in r.tflops), r
        assert not r.flags & (N.CT_ECC | N.CT_ECC_CORRECTED), r
        if not _gpu_busy():
            assert r.sms_covered == r.sm_count, r
        assert abs(free1 - free0) < 2 * MiB, (free0, free1)
        (p,) = ctx.probe_health(min_gbs=1e-3)
        assert p.healthy and not p.flags & N.RES_COMPUTE
    print("L2 test 100 ms/format: SMs %d/%d, ms %s, TB/s word %.2f byte %.2f, G ops/s atom %.2f"
          % (r.sms_covered, r.sm_count, ["%.1f" % x for x in r.ms], *r.tflops))


def test_l2_test_fault_is_attributed_and_latched_until_reset(pkg):
    N = pkg._native
    with _open(pkg) as ctx:
        (r,) = ctx.l2_test(0, duration_ms=10, fault_sm=0, fault_mask=0x10)
        assert not r.healthy and r.err == 0, r
        assert r.mismatches == [1, 1, 1], r
        assert r.first_bad_format == N.L2_WORD and r.first_bad_tile == 0 and len(r.bad_sms()) >= 1, r
        (p,) = ctx.probe_health(min_gbs=1e-3)
        assert p.flags & N.RES_COMPUTE and not p.healthy
        ctx.probe_reset(0)
        (p,) = ctx.probe_health(min_gbs=1e-3)
        assert p.healthy and not p.flags & N.RES_COMPUTE


def test_l2_test_skips_a_busy_gpu(pkg):
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
            (r,) = ctx.l2_test(0, duration_ms=10, fault_sm=0, fault_mask=1)
            assert r.flags & N.CT_SKIPPED_BUSY and r.mismatches == [0, 0, 0] and r.ms == [0, 0, 0], r
            (r,) = ctx.l2_test(0, duration_ms=10, even_if_busy=True)
            assert not r.flags & N.CT_SKIPPED_BUSY and r.healthy and r.err == 0, r
    finally:
        if helper.poll() is None:
            helper.kill()
        helper.wait()


def test_daemon_l2_test_at_start_logs_a_clean_result(short_dir):
    exe = os.path.join(ROOT, "k8s-device-plugin_b200", "b200dp_plugind")
    proc = subprocess.Popen([exe, "-backend=cuda:devices=0,bytes=67108864,calib=1", "-plugin_dir", short_dir,
                             "-start_retry_wait=0.05", "-l2_test_at_start=2", "-compute_test_ms=50"],
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
    assert log.index("L2 test ") < log.index("Failed to start plugin"), log[-3000:]
    got = [ln for ln in log.splitlines() if ln.startswith("L2 test ")]
    assert len(got) == 1 and ": Healthy, flags 0x" in got[0] and "mismatches 0/0/0, first bad SM -1" in got[0], log[-3000:]
