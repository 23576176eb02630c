"""GPU tests of the on-demand register-file self-test (b2dp_regfile_test, csrc/rf_selftest.cuh).

Through tests/native/libregfile_test_kernels_test.so (the kernel launched directly, one format at a time):
  - cudaOccupancyMaxActiveBlocksPerMultiprocessor gives two CTAs per SM, and every SM id runs two;
  - the DUMP instantiation's final registers, every thread's fold and OR of direct-compare differences equal
    tests/rf_test_oracle.py bit for bit, in every format, tile and CTA;
  - a flip at a chosen thread, register and element is counted in exactly the first comparison, by exactly the CTA on
    the chosen SM.
Through the ABI: a clean run, fault attribution, the latch and b2dp_probe_reset, the busy skip, and the daemon's
start-up test.
"""
import ctypes as C
import os
import signal
import subprocess
import sys
import time

import numpy as np
import pytest

import rf_test_oracle as ro

pytestmark = pytest.mark.gpu

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(HERE)
LIB_PATH = os.path.join(HERE, "native", "libregfile_test_kernels_test.so")
MiB = 1 << 20
MS = 1000000
FMT_IDS = [ro.NAMES[f] for f in ro.FORMATS]
_P = C.POINTER


class CtRecord(C.Structure):
    _fields_ = [("smid", C.c_uint32), ("nsmid", C.c_uint32), ("rounds", C.c_uint64), ("comparisons", C.c_uint64),
                ("mismatches", C.c_uint64), ("first_bad_tile", C.c_int32), ("first_bad_rep", C.c_int32),
                ("seq", C.c_uint64)]


class Harness:
    def __init__(self, device=0):
        L = C.CDLL(LIB_PATH)
        L.rf_open.restype = C.c_void_p
        L.rf_open.argtypes = [C.c_int, C.c_char_p, C.c_int]
        L.rf_close.argtypes = [C.c_void_p]
        L.rf_error.restype = C.c_char_p
        L.rf_error.argtypes = [C.c_void_p]
        L.rf_sms.argtypes = [C.c_void_p]
        L.rf_grid.argtypes = [C.c_void_p, C.c_int]
        L.rf_per_sm.argtypes = [C.c_void_p, C.c_int]
        L.rf_dump.argtypes = [C.c_void_p, C.c_int, C.c_uint32, C.c_uint32, C.c_uint32, C.c_uint32, C.c_int, C.c_uint32,
                              _P(C.c_uint32), _P(CtRecord), C.c_int, _P(C.c_int), _P(C.c_float)]
        L.rf_run.argtypes = [C.c_void_p, C.c_int, C.c_uint32, C.c_uint64, C.c_uint32, C.c_uint32, C.c_uint32, C.c_int,
                             C.c_uint32, _P(CtRecord), C.c_int, _P(C.c_int), _P(C.c_float)]
        assert L.rf_record_bytes() == C.sizeof(CtRecord)
        assert L.rf_dump_words() == ro.DUMP_WORDS and L.rf_held() == ro.HELD
        self.L = L
        err = C.create_string_buffer(512)
        self.h = L.rf_open(device, err, len(err))
        if not self.h:
            raise RuntimeError("rf_open: " + err.value.decode())
        self.sms = L.rf_sms(self.h)

    def close(self):
        if self.h:
            self.L.rf_close(self.h)
            self.h = None

    def _check(self, rc, what):
        if rc == 1:
            raise RuntimeError("%s: %s" % (what, self.L.rf_error(self.h).decode()))
        assert rc == 0, "%s refused: code %d" % (what, rc)

    def grid(self, fmt):
        return self.L.rf_grid(self.h, fmt)

    def dump(self, fmt, seed):
        g = self.grid(fmt)
        out = np.zeros((g, ro.TILES, ro.DUMP_WORDS), dtype=np.uint32)
        recs = (CtRecord * g)()
        n, ms = C.c_int(), C.c_float()
        self._check(self.L.rf_dump(self.h, fmt, seed, ro.HOOK_REG, ro.HOOK_ELEMENT, ro.HOOK_THREAD, -1, 0,
                                   out.ctypes.data_as(_P(C.c_uint32)), recs, g, C.byref(n), C.byref(ms)), "rf_dump")
        return out, list(recs[:n.value]), ms.value

    def run(self, fmt, seed, duration_ms, hook=(ro.HOOK_REG, ro.HOOK_ELEMENT, ro.HOOK_THREAD), fault_sm=-1,
            fault_mask=0):
        g = self.grid(fmt)
        recs = (CtRecord * g)()
        n, ms = C.c_int(), C.c_float()
        self._check(self.L.rf_run(self.h, fmt, seed, int(duration_ms * MS), hook[0], hook[1], hook[2], fault_sm,
                                  fault_mask, recs, g, C.byref(n), C.byref(ms)), "rf_run")
        return list(recs[:n.value]), ms.value


@pytest.fixture(scope="module")
def H():
    if not os.path.exists(LIB_PATH):
        pytest.skip("run __graft_entry__.build() first")
    h = Harness(0)
    yield h
    h.close()


def _arrived(recs, seq=7):
    for r in recs:
        assert r.seq == seq and r.rounds >= 1 and r.comparisons == r.rounds * ro.TILES * ro.REPS, \
            (r.smid, r.seq, r.rounds, r.comparisons)
        assert r.smid < r.nsmid <= 256


def _check_clean(recs):
    _arrived(recs)
    for r in recs:
        assert r.mismatches == 0 and (r.first_bad_tile, r.first_bad_rep) == (-1, -1), (r.smid, r.mismatches)


# ---- the kernel against the oracle --------------------------------------------------------------------------------
def test_two_ctas_on_every_sm(H):
    regs = [H.L.rf_num_regs(f, 0) for f in ro.FORMATS]
    print("regfile test: %d SMs, CTAs per SM %s, registers per thread %s"
          % (H.sms, [H.L.rf_per_sm(H.h, f) for f in ro.FORMATS], regs))
    for fmt in ro.FORMATS:
        assert H.L.rf_per_sm(H.h, fmt) == 2, fmt
        assert H.grid(fmt) == 2 * H.sms
    recs, _ = H.run(ro.ALU, 1, 0)
    _check_clean(recs)
    ids = sorted(r.smid for r in recs)
    assert len(set(ids)) == H.sms and all(ids.count(s) == 2 for s in set(ids)), ids


@pytest.mark.parametrize("fmt", ro.FORMATS, ids=FMT_IDS)
def test_dump_equals_the_oracle(H, fmt):
    seed = 0xC0FFEE17
    d, recs, _ = H.dump(fmt, seed)
    _check_clean(recs)
    assert all(r.rounds == 1 for r in recs)
    for t in range(ro.TILES):
        want = ro.march(fmt, ro.kind(t), ro.key(seed, fmt, t))
        regs = want["regs"].T.ravel()                        # register j of thread t at word j * THREADS + t
        for cta in range(len(recs)):
            got = d[cta, t]
            n = ro.HELD * ro.THREADS
            assert np.array_equal(got[:n], regs), (t, cta, np.argwhere(got[:n] != regs)[:4].ravel())
            assert np.array_equal(got[n:n + ro.THREADS], want["fold"]), (t, cta)
            assert not got[n + ro.THREADS:].any(), (t, cta)


FAULT_THREADS = [0, 31, 64, 127]
FAULT_REGS = [0, ro.HELD // 2, ro.HELD - 1]


@pytest.mark.parametrize("fmt", ro.FORMATS, ids=FMT_IDS)
def test_flip_is_counted_in_exactly_its_comparison_by_exactly_its_cta(H, fmt):
    recs, _ = H.run(fmt, 3, 0)
    _check_clean(recs)
    smids = [r.smid for r in recs]
    targets = [0, len(recs) // 2 + 1, len(recs) - 1]
    n = 0
    for e in range(ro.ELEMENTS[fmt] - 1):
        for th in FAULT_THREADS:
            for j in FAULT_REGS:
                for mask in (0x1, 0x80000000, 0xFFFFFFFF):
                    s = smids[targets[n % len(targets)]]
                    n += 1
                    got, _ = H.run(fmt, 3, 0, hook=(j, e, th), fault_sm=s, fault_mask=mask)
                    _arrived(got)
                    # both CTAs on SM s carry the hook: each counts exactly the first comparison
                    for i, r in enumerate(got):
                        want = (1, 0, 0) if r.smid == s else (0, -1, -1)
                        assert (r.mismatches, r.first_bad_tile, r.first_bad_rep) == want, \
                            (e, th, j, hex(mask), i, r.smid, s)


# ---- through the ABI ----------------------------------------------------------------------------------------------
def _open(pkg, nbytes=64 * MiB):
    return pkg.Context("cuda:devices=0,bytes=%d,calib=1" % nbytes)


def _card():
    try:
        out = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader",
                              "-i", "0"], capture_output=True, text=True, timeout=30).stdout.strip()
    except Exception as e:       # noqa: BLE001
        out = "nvidia-smi unavailable: %s" % e
    return out


def test_regfile_test_clean(pkg, H):
    import torch
    torch.cuda.init()
    N = pkg._native
    with _open(pkg) as ctx:
        ctx.regfile_test(0, duration_ms=10)                    # first launch loads the kernels: not counted below
        (r,) = ctx.regfile_test(0, duration_ms=300)
        assert r.healthy and r.err == 0, r
        assert r.mismatches == [0, 0, 0] and r.bad_sm_mask == [0, 0, 0, 0], r
        assert not r.flags & N.CT_ECC, r
        assert (r.first_bad_sm, r.first_bad_format, r.first_bad_tile) == (-1, -1, -1)
        assert r.sm_count == torch.cuda.get_device_properties(0).multi_processor_count == H.sms
        assert r.sms_covered == r.sm_count and not r.flags & N.CT_PARTIAL_COVERAGE, r
        assert all(ms >= 290 for ms in r.ms) and all(t > 0 for t in r.tflops), r
        (p,) = ctx.probe_health(min_gbs=1e-3)
        assert p.healthy and not p.flags & N.RES_COMPUTE
    print("regfile test 300 ms/format on %s: flags 0x%x, SMs %d/%d, ms %s, TB/s alu %.2f load %.2f hold %.2f"
          % (_card(), r.flags, r.sms_covered, r.sm_count, ["%.1f" % x for x in r.ms], *r.tflops))


@pytest.mark.parametrize("where", ["first", "middle", "last"])
def test_regfile_test_fault_is_attributed_and_latched_until_reset(pkg, H, where):
    N = pkg._native
    recs, _ = H.run(ro.ALU, 1, 0)
    ids = sorted({r.smid for r in recs})
    s = {"first": ids[0], "middle": ids[len(ids) // 2], "last": ids[-1]}[where]
    with _open(pkg) as ctx:
        (r,) = ctx.regfile_test(0, duration_ms=10, fault_sm=s, fault_mask=0x80000000)
        assert not r.healthy and r.err == 0, r
        assert r.bad_sms() == [s] and (r.first_bad_sm, r.first_bad_tile) == (s, 0), r
        # every format: the hook flips the register in both CTAs on the SM, each counts its first comparison
        assert r.first_bad_format == N.RF_ALU and r.mismatches == [2, 2, 2], r
        (p,) = ctx.probe_health(min_gbs=1e-3)
        assert p.flags & N.RES_COMPUTE and not p.healthy and p.mismatches == 0
        ctx.probe_reset(0)
        (p,) = ctx.probe_health(min_gbs=1e-3)
        assert p.healthy and not p.flags & N.RES_COMPUTE
        (r,) = ctx.regfile_test(0, duration_ms=10)
        assert r.healthy and r.bad_sm_mask == [0, 0, 0, 0], r


def test_regfile_test_skips_a_busy_gpu(pkg):
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
            (r,) = ctx.regfile_test(0, duration_ms=10, fault_sm=0, fault_mask=1)
            assert r.flags & N.CT_SKIPPED_BUSY and r.mismatches == [0, 0, 0] and r.ms == [0, 0, 0], r
            (p,) = ctx.probe_health(min_gbs=1e-3)
            assert not p.flags & N.RES_COMPUTE
            (r,) = ctx.regfile_test(0, duration_ms=10, even_if_busy=True)
            assert not r.flags & N.CT_SKIPPED_BUSY and r.healthy and r.err == 0, r
    finally:
        if helper.poll() is None:
            helper.kill()
        helper.wait()


def test_daemon_regfile_test_at_start_logs_a_clean_result(short_dir):
    exe = os.path.join(ROOT, "k8s-device-plugin_b200", "b200dp_plugind")

    def lines(level):
        proc = subprocess.Popen([exe, "-backend=cuda:devices=0,bytes=67108864,calib=1", "-plugin_dir", short_dir,
                                 "-start_retry_wait=0.05", "-regfile_test_at_start=%d" % level, "-compute_test_ms=50"],
                                stderr=subprocess.PIPE, text=True)
        got = []
        try:
            t0 = time.time()
            while time.time() - t0 < 120:
                line = proc.stderr.readline()
                if not line:
                    break
                got.append(line)
                if "Failed to start plugin" in line:
                    break
        finally:
            proc.send_signal(signal.SIGINT)
            rest = proc.communicate(timeout=30)[1]
        log = "".join(got) + rest
        assert proc.returncode == 0, log[-3000:]
        assert log.index("regfile test ") < log.index("Failed to start plugin"), log[-3000:]
        return [ln for ln in log.splitlines() if ln.startswith("regfile test ")], log

    got, log = lines(1)
    assert len(got) == 1, log[-3000:]
    if "flags 0x1," in got[0]:
        got, log = lines(2)
        assert len(got) == 1, log[-3000:]
    assert ": Healthy, flags 0x" in got[0] and "mismatches 0/0/0, first bad SM -1" in got[0], log[-3000:]
