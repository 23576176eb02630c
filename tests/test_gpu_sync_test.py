"""The on-demand synchronization self-test on a real H100.

- The kernel of sync_selftest.cuh, launched directly (tests/native/libsync_test_kernels_test.so):
  - the DUMP instantiation's result words equal the host reference (sync_test_math.hpp through
    tests/native/sync_test_math_test.cpp) word for word, for every format and tile at two seeds;
  - a clean run covers every SM id and every CTA compares exactly what its rounds hold, at 32 seeds per format;
  - on caller-built tables, a wrong check value in any of the 128 threads is counted in exactly its tile's repetitions,
    and check values computed by each fault model of tests/sync_test_oracle.py mismatch in every tile and repetition;
  - malformed tables are refused before anything runs.
- b2dp_sync_test through the ABI: Healthy on an idle card with free memory back where it started, the fault hook at the
  first, a middle and the last SM attributed to its SM and latched (RES_COMPUTE) until probe_reset, the busy skip,
  and the daemon's -sync_test_at_start.

Every run is short: 0-100 ms per format."""
import ctypes as C
import os
import shutil
import subprocess
import sys

import numpy as np
import pytest

import sync_test_oracle as so

pytestmark = pytest.mark.gpu

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(HERE)
CSRC = os.path.join(ROOT, "k8s-device-plugin_b200", "csrc")
LIB_PATH = os.path.join(HERE, "native", "libsync_test_kernels_test.so")
MS = 1000000
MiB = 1 << 20
TILES, REPS, THREADS = 8, 16, 128
FORMATS = (0, 1, 2)
FMT_IDS = ["atom", "bar", "warp"]


class CtRecord(C.Structure):
    _fields_ = [("smid", C.c_uint32), ("nsmid", C.c_uint32), ("rounds", C.c_uint64), ("comparisons", C.c_uint64),
                ("mismatches", C.c_uint64), ("first_bad_tile", C.c_int32), ("first_bad_rep", C.c_int32),
                ("seq", C.c_uint64)]


_P = C.POINTER


class Ref:
    """tests/native/sync_test_math_test.cpp: tables, result words and checks of the host reference."""

    def __init__(self, exe):
        self.p = subprocess.Popen([exe], stdin=subprocess.PIPE, stdout=subprocess.PIPE, text=True)
        self.p.stdin.write("bounds\n")
        self.p.stdin.flush()
        b = [float(x) for x in self.p.stdout.readline().split()]
        self.slots = [int(b[4 * f]) for f in FORMATS]
        self.words = [int(b[4 * f + 1]) for f in FORMATS]

    def tile(self, seed, fmt, tile):
        self.p.stdin.write("tile %d %d %d\n" % (seed, fmt, tile))
        self.p.stdin.flush()
        v = np.array([int(x) for x in self.p.stdout.readline().split()], dtype=np.uint64).astype(np.uint32)
        ns, nw = self.slots[fmt] * THREADS, self.words[fmt] * THREADS
        return v[:ns], v[ns:ns + nw].reshape(THREADS, -1), v[ns + nw:]

    def launch_tables(self, seed, fmt):
        tabs, words, checks = zip(*(self.tile(seed, fmt, t) for t in range(TILES)))
        return np.concatenate(tabs), np.stack(words), np.stack(checks)

    def close(self):
        self.p.stdin.close()
        self.p.wait()


@pytest.fixture(scope="module")
def ref(tmp_path_factory):
    exe = str(tmp_path_factory.mktemp("sy") / "sync_test_math_test")
    subprocess.run(["g++", "-O2", "-std=c++17", "-I", CSRC, os.path.join(HERE, "native", "sync_test_math_test.cpp"),
                    "-o", exe], check=True)
    r = Ref(exe)
    yield r
    r.close()


class Harness:
    def __init__(self, device=0):
        L = C.CDLL(LIB_PATH)
        L.sk_open.restype = C.c_void_p
        L.sk_open.argtypes = [C.c_int, C.c_char_p, C.c_int]
        L.sk_close.argtypes = [C.c_void_p]
        L.sk_error.restype = C.c_char_p
        L.sk_error.argtypes = [C.c_void_p]
        L.sk_sms.argtypes = [C.c_void_p]
        L.sk_table_bytes.restype = C.c_uint64
        L.sk_occupancy.argtypes = [C.c_void_p, C.c_int, _P(C.c_int)]
        L.sk_dump.argtypes = [C.c_void_p, C.c_int, C.c_uint32, _P(C.c_uint32), _P(CtRecord)]
        L.sk_run.argtypes = [C.c_void_p, C.c_int, C.c_uint32, C.c_uint64, C.c_int, C.c_uint32, _P(CtRecord), C.c_int,
                             _P(C.c_int), _P(C.c_float)]
        L.sk_run_tables.argtypes = [C.c_void_p, C.c_int, C.c_int, C.c_void_p, C.c_uint64, C.c_void_p, C.c_uint64,
                                    C.c_int, C.c_uint64, _P(CtRecord), C.c_int, _P(C.c_int), _P(C.c_float),
                                    _P(C.c_uint32)]
        assert L.sk_record_bytes() == C.sizeof(CtRecord)
        self.L = L
        err = C.create_string_buffer(512)
        self.h = L.sk_open(device, err, len(err))
        if not self.h:
            raise RuntimeError("sk_open: " + err.value.decode())
        self.sms = L.sk_sms(self.h)

    def close(self):
        if self.h:
            self.L.sk_close(self.h)
            self.h = None

    def _check(self, rc, what):
        if rc == 1:
            raise RuntimeError("%s: %s" % (what, self.L.sk_error(self.h).decode()))
        assert rc == 0, "%s refused: code %d" % (what, rc)

    def occupancy(self, fmt):
        n = C.c_int()
        self._check(self.L.sk_occupancy(self.h, fmt, C.byref(n)), "sk_occupancy")
        return n.value

    def dump(self, fmt, seed):
        words = self.L.sk_words(fmt)
        out = np.zeros(TILES * THREADS * words, dtype=np.uint32)
        rec = CtRecord()
        self._check(self.L.sk_dump(self.h, fmt, seed, out.ctypes.data_as(_P(C.c_uint32)), C.byref(rec)), "sk_dump")
        return out.reshape(TILES, THREADS, words), rec

    def run(self, fmt, seed, duration_ms, fault_sm=-1, fault_mask=0):
        cap = self.sms * 32
        recs = (CtRecord * cap)()
        n, ms = C.c_int(), C.c_float()
        self._check(self.L.sk_run(self.h, fmt, seed, int(duration_ms * MS), fault_sm, fault_mask, recs, cap,
                                  C.byref(n), C.byref(ms)), "sk_run")
        return list(recs[:n.value]), ms.value

    def run_tables_rc(self, fmt, tables, checks, grid=1, duration_ms=0, table_bytes=None, n_checks=None):
        cap = max(grid, 1)
        recs = (CtRecord * cap)()
        n, ms = C.c_int(), C.c_float()
        rc = self.L.sk_run_tables(self.h, fmt, 0, tables.ctypes.data, tables.nbytes if table_bytes is None
                                  else table_bytes, checks.ctypes.data, checks.size if n_checks is None else n_checks,
                                  grid, int(duration_ms * MS), recs, cap, C.byref(n), C.byref(ms), None)
        return rc, list(recs[:n.value]) if rc == 0 else []


@pytest.fixture(scope="module")
def H():
    if not os.path.exists(LIB_PATH):
        pytest.skip("run __graft_entry__.build() first")
    h = Harness(0)
    yield h
    h.close()


def _complete(r, seq_ok=True):
    return r.rounds >= 1 and r.comparisons == r.rounds * TILES * REPS


@pytest.mark.parametrize("fmt", FORMATS, ids=FMT_IDS)
@pytest.mark.parametrize("seed", [1, 0xC0FFEE])
def test_dump_equals_reference(H, ref, fmt, seed):
    got, rec = H.dump(fmt, seed)
    _, want, _ = ref.launch_tables(seed, fmt)
    bad = np.argwhere(got != want)
    assert bad.size == 0, "first differing (tile, thread, word): %s got %#x want %#x (%d words differ)" % (
        tuple(bad[0]), got[tuple(bad[0])], want[tuple(bad[0])], len(bad))
    assert rec.mismatches == 0 and _complete(rec)


@pytest.mark.parametrize("fmt", FORMATS, ids=FMT_IDS)
def test_clean_runs_cover_every_sm(H, fmt):
    seen = set()
    for seed in range(32):
        recs, _ = H.run(fmt, 0x5EED0000 + seed, 0 if seed else 100)
        assert len(recs) == H.sms * H.occupancy(fmt)
        for r in recs:
            assert _complete(r) and r.mismatches == 0, (seed, r.smid, r.rounds, r.comparisons, r.mismatches)
            seen.add(r.smid)
    assert len(seen) == H.sms


@pytest.mark.parametrize("fmt", FORMATS, ids=FMT_IDS)
def test_wrong_check_counted_in_its_tile(H, ref, fmt):
    tables, _, checks = ref.launch_tables(7, fmt)
    for t in (0, 37, 127):
        tile = t % TILES
        c = checks.copy()
        c[tile, t] ^= 1 << (t % 32)
        recs = H.run_tables_rc(fmt, tables, c, grid=2)[1]
        for r in recs:
            assert r.rounds == 1 and r.comparisons == TILES * REPS
            assert r.mismatches == REPS and r.first_bad_tile == tile and r.first_bad_rep == 0


@pytest.mark.parametrize("fmt", FORMATS, ids=FMT_IDS)
def test_malformed_tables_refused(H, ref, fmt):
    tables, _, checks = ref.launch_tables(3, fmt)
    assert H.run_tables_rc(fmt, tables, checks, table_bytes=tables.nbytes - 4)[0] not in (0, 1)
    assert H.run_tables_rc(fmt, tables, checks, n_checks=checks.size - 1)[0] not in (0, 1)
    assert H.run_tables_rc(fmt, tables, checks, grid=0)[0] not in (0, 1)


@pytest.mark.parametrize("fmt,fault", [(f, m) for f in FORMATS for m in so.FAULTS[f]])
def test_fault_model_checks_mismatch_in_every_tile(H, fmt, fault):
    """Check values a device with the fault would match: this healthy H100 mismatches them in every tile and
    repetition, and only there (the table is the oracle's, which equals the C++)."""
    seed = 0xFA17
    tables = np.concatenate([np.array(so.table(seed, fmt, t), dtype=np.uint64).astype(np.uint32).ravel()
                             for t in range(TILES)])
    checks = np.array([so.checks(seed, fmt, t, fault=fault) for t in range(TILES)], dtype=np.uint64).astype(np.uint32)
    clean = np.array([so.checks(seed, fmt, t) for t in range(TILES)], dtype=np.uint64).astype(np.uint32)
    rc, recs = H.run_tables_rc(fmt, tables, checks, grid=1)
    assert rc == 0 and len(recs) == 1
    r = recs[0]
    assert r.rounds == 1 and r.comparisons == TILES * REPS
    assert r.mismatches == TILES * REPS and (r.first_bad_tile, r.first_bad_rep) == (0, 0), (fault, r.mismatches)
    rc, recs = H.run_tables_rc(fmt, tables, clean, grid=1)
    assert rc == 0 and recs[0].mismatches == 0


# ---- through the ABI ---------------------------------------------------------------------------------------------------
@pytest.fixture(scope="module")
def pkg():
    sys.path.insert(0, ROOT)
    import importlib
    return importlib.import_module("k8s-device-plugin_b200")


def _open(pkg, nbytes=64 * MiB):
    return pkg.Context("cuda:devices=0,bytes=%d,calib=1" % nbytes)


def _gpu_busy():
    """True if NVML lists a compute process on GPU 0 besides this one (the rule b2dp_sync_test applies)."""
    try:
        import pynvml
        pynvml.nvmlInit()
        return len(pynvml.nvmlDeviceGetComputeRunningProcesses(pynvml.nvmlDeviceGetHandleByIndex(0))) > 1
    except Exception:       # noqa: BLE001
        return None


@pytest.fixture(scope="module")
def sm_ids(H):
    recs, _ = H.run(1, 0x5EED, 20)
    assert all(_complete(r) and r.mismatches == 0 for r in recs)
    return sorted({r.smid for r in recs})


def test_sync_test_clean_and_memory_back(pkg):
    import torch
    torch.cuda.init()
    N = pkg._native
    with _open(pkg) as ctx:
        ctx.sync_test(0, duration_ms=10)                        # first launch loads the kernels: not counted below
        free0, _ = torch.cuda.mem_get_info(0)
        (r,) = ctx.sync_test(0, duration_ms=100)
        free1, _ = torch.cuda.mem_get_info(0)
        assert r.healthy and r.err == 0, r
        assert r.mismatches == [0, 0, 0] and r.bad_sm_mask == [0, 0, 0, 0], r
        assert (r.first_bad_sm, r.first_bad_format, r.first_bad_tile) == (-1, -1, -1)
        assert r.sm_count == torch.cuda.get_device_properties(0).multi_processor_count
        assert all(ms >= 90 for ms in r.ms) and all(t > 0 for t in r.tflops), r
        if not _gpu_busy():
            assert r.sms_covered == r.sm_count and r.flags == 0, r
        assert abs(free1 - free0) < 2 * MiB, (free0, free1)
        (p,) = ctx.probe_health(min_gbs=1e-3)
        assert p.healthy and not p.flags & N.RES_COMPUTE


@pytest.mark.parametrize("where,mask", [("first", 0x1), ("middle", 0x80000000), ("last", 0xFFFFFFFF)])
def test_sync_test_fault_is_attributed_and_latched_until_reset(pkg, H, sm_ids, where, mask):
    N = pkg._native
    s = {"first": sm_ids[0], "middle": sm_ids[len(sm_ids) // 2], "last": sm_ids[-1]}[where]
    with _open(pkg) as ctx:
        (r,) = ctx.sync_test(0, duration_ms=10, fault_sm=s, fault_mask=mask)
        assert not r.healthy and r.err == 0, r
        assert r.bad_sms() == [s], r.bad_sms()
        assert (r.first_bad_sm, r.first_bad_format, r.first_bad_tile) == (s, N.SY_ATOM, 0), r
        for f in FORMATS:          # one mismatch per CTA that ran on s
            assert 1 <= r.mismatches[f] <= H.occupancy(f), (f, r.mismatches)
        (p,) = ctx.probe_health(min_gbs=1e-3)
        assert p.flags & N.RES_COMPUTE and not p.healthy and p.mismatches == 0
        ctx.probe_reset(0)
        (p,) = ctx.probe_health(min_gbs=1e-3)
        assert p.healthy and not p.flags & N.RES_COMPUTE


def test_sync_test_skips_a_busy_gpu(pkg):
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
            (r,) = ctx.sync_test(0, duration_ms=10, fault_sm=0, fault_mask=1)
            assert r.flags & N.CT_SKIPPED_BUSY and r.mismatches == [0, 0, 0] and r.ms == [0, 0, 0], r
            (p,) = ctx.probe_health(min_gbs=1e-3)
            assert not p.flags & N.RES_COMPUTE
            (r,) = ctx.sync_test(0, duration_ms=10, even_if_busy=True)
            assert not r.flags & N.CT_SKIPPED_BUSY and r.healthy and r.err == 0, r
    finally:
        if helper.poll() is None:
            helper.kill()
        helper.wait()


def test_daemon_sync_test_at_start(tmp_path):
    exe = os.path.join(ROOT, "k8s-device-plugin_b200", "b200dp_plugind")
    if not os.path.exists(exe):
        pytest.skip("no daemon build")
    d = tmp_path / "p"
    d.mkdir()
    proc = subprocess.Popen([exe, "-backend=cuda:devices=0,bytes=67108864,calib=1", "-plugin_dir", str(d), "-start_retry_wait=0.05",
                             "-sync_test_at_start=1", "-compute_test_ms=50"], stderr=subprocess.PIPE, text=True)
    line = ""
    try:
        for _ in range(200):
            line = proc.stderr.readline()
            if "sync test" in line or not line:
                break
    finally:
        proc.terminate()
        try:
            proc.wait(timeout=10)
        except subprocess.TimeoutExpired:
            proc.kill()
            proc.wait()
    assert "sync test" in line and "Healthy" in line and "Unhealthy" not in line, line
