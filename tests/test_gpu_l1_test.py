"""The on-demand L1 self-test on a real H100.

- The kernel of l1_selftest.cuh, launched directly (tests/native/libl1_test_kernels_test.so):
  - the DUMP instantiation's values equal the host reference (l1_test_math.hpp through tests/native/l1_test_math_test.cpp)
    word for word, for every format and tile at two seeds: the raw span words of L1_DATA, every texel fetch, gather and
    address mode of L1_TEX, every constant load of L1_CONST;
  - a clean run covers every SM id, every CTA compares exactly what its rounds hold, and on an idle card every SM id
    carries exactly the occupancy's number of CTAs;
  - on caller-built tables, a wrong check value in any thread is counted in exactly its tile's repetitions, and check
    values computed by the fault models of tests/l1_test_oracle.py mismatch where the model says they must;
  - malformed tables, out-of-range indices and a zero texture handle are refused before anything launches.
- b2dp_l1_test through the ABI: Healthy on an idle card with free memory back where it started (the CUDA array
  included), the fault hook at the first, a middle and the last SM attributed to its SM and latched (RES_COMPUTE) until
  probe_reset, the busy skip, and the daemon's -l1_test_at_start.

Every run is short: 0-100 ms per format."""
import ctypes as C
import os
import subprocess
import sys

import numpy as np
import pytest

import l1_test_oracle as lo

pytestmark = pytest.mark.gpu

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(HERE)
CSRC = os.path.join(ROOT, "k8s-device-plugin_b200", "csrc")
LIB_PATH = os.path.join(HERE, "native", "libl1_test_kernels_test.so")
MS = 1000000
MiB = 1 << 20
TILES, REPS, THREADS = 8, 16, 128
FORMATS = (0, 1, 2)
FMT_IDS = ["data", "tex", "const"]
TEX_OPS = ["tld", "tex", "wrap", "mirror", "clamp", "border", "tld4", "ld.nc"]


class CtRecord(C.Structure):
    _fields_ = [("smid", C.c_uint32), ("nsmid", C.c_uint32), ("rounds", C.c_uint64), ("comparisons", C.c_uint64),
                ("mismatches", C.c_uint64), ("first_bad_tile", C.c_int32), ("first_bad_rep", C.c_int32),
                ("seq", C.c_uint64)]


_P = C.POINTER


class Ref:
    """tests/native/l1_test_math_test.cpp: tables, result words, checks and L1_DATA's raw reads of the host reference."""

    def __init__(self, exe):
        self.p = subprocess.Popen([exe], stdin=subprocess.PIPE, stdout=subprocess.PIPE, text=True)
        b = [float(x) for x in self.ask("bounds").split()]
        self.words = [int(b[3 * f]) for f in FORMATS]

    def ask(self, q):
        self.p.stdin.write(q + "\n")
        self.p.stdin.flush()
        return self.p.stdout.readline()

    def _arr(self, q):
        return np.array(self.ask(q).split(), dtype=np.uint64).astype(np.uint32)

    def tile(self, seed, fmt, tile):
        v = self._arr("tile %d %d %d" % (seed, fmt, tile))
        nw = self.words[fmt] * THREADS
        return v[:4], v[4:4 + nw].reshape(THREADS, -1), v[4 + nw:]

    def span(self, seed, tile, K, c=0):
        return self._arr("span %d %d %d %d" % (seed, tile, K, c)).reshape(THREADS, -1)

    def launch_tables(self, seed, fmt):
        tabs, words, checks = zip(*(self.tile(seed, fmt, t) for t in range(TILES)))
        return np.concatenate(tabs), np.stack(words), np.stack(checks)

    def close(self):
        self.p.stdin.close()
        self.p.wait()


@pytest.fixture(scope="module")
def ref(tmp_path_factory):
    exe = str(tmp_path_factory.mktemp("l1") / "l1_test_math_test")
    subprocess.run(["g++", "-O2", "-std=c++17", "-I", CSRC, os.path.join(HERE, "native", "l1_test_math_test.cpp"),
                    "-o", exe], check=True)
    r = Ref(exe)
    yield r
    r.close()


class Harness:
    def __init__(self, device=0):
        L = C.CDLL(LIB_PATH)
        L.l1k_open.restype = C.c_void_p
        L.l1k_open.argtypes = [C.c_int, C.c_char_p, C.c_int]
        L.l1k_close.argtypes = [C.c_void_p]
        L.l1k_error.restype = C.c_char_p
        L.l1k_error.argtypes = [C.c_void_p]
        L.l1k_sms.argtypes = [C.c_void_p]
        L.l1k_occupancy.argtypes = [C.c_void_p, C.c_int, C.c_int, _P(C.c_int)]
        L.l1k_default_blocks.argtypes = [C.c_void_p, _P(C.c_uint)]
        L.l1k_dump_words.restype = C.c_uint64
        L.l1k_dump_words.argtypes = [C.c_int, C.c_uint]
        L.l1k_run.argtypes = [C.c_void_p, C.c_int, C.c_int, C.c_uint32, C.c_uint, C.c_int, C.c_uint64, C.c_int,
                              C.c_uint32, _P(CtRecord), C.c_int, _P(C.c_int), _P(C.c_float), _P(C.c_uint),
                              _P(C.c_uint32)]
        L.l1k_run_tables.argtypes = [C.c_void_p, C.c_int, C.c_uint32, C.c_void_p, C.c_uint64, C.c_void_p, C.c_uint64,
                                     C.c_int, C.c_uint, C.c_uint64, C.c_int, _P(CtRecord), C.c_int, _P(C.c_int),
                                     _P(C.c_float)]
        assert L.l1k_record_bytes() == C.sizeof(CtRecord)
        self.L = L
        err = C.create_string_buffer(512)
        self.h = L.l1k_open(device, err, len(err))
        if not self.h:
            raise RuntimeError("l1k_open: " + err.value.decode())
        self.sms = L.l1k_sms(self.h)

    def close(self):
        if self.h:
            self.L.l1k_close(self.h)
            self.h = None

    def _check(self, rc, what):
        if rc == 1:
            raise RuntimeError("%s: %s" % (what, self.L.l1k_error(self.h).decode()))
        assert rc == 0, "%s refused: code %d" % (what, rc)

    def occupancy(self, fmt):
        n = C.c_int()
        self._check(self.L.l1k_occupancy(self.h, fmt, 0, C.byref(n)), "l1k_occupancy")
        return n.value

    def default_blocks(self):
        k = C.c_uint()
        self._check(self.L.l1k_default_blocks(self.h, C.byref(k)), "l1k_default_blocks")
        return k.value

    def run(self, fmt, seed, duration_ms, K=0, carveout=0, fault_sm=-1, fault_mask=0, dump=False):
        """Every CTA's record, the launch's ms, the K used, and with dump the DUMP words (CTA 0 alone)."""
        cap = self.sms * 32
        recs = (CtRecord * cap)()
        n, ms, k = C.c_int(), C.c_float(), C.c_uint()
        out = None
        if dump:
            kd = K or self.default_blocks()
            out = np.zeros(self.L.l1k_dump_words(fmt, kd), dtype=np.uint32)
        self._check(self.L.l1k_run(self.h, fmt, int(dump), seed, K, carveout, int(duration_ms * MS), fault_sm,
                                   fault_mask, recs, cap, C.byref(n), C.byref(ms), C.byref(k),
                                   out.ctypes.data_as(_P(C.c_uint32)) if dump else None), "l1k_run")
        return list(recs[:n.value]), ms.value, k.value, out

    def run_tables_rc(self, fmt, seed, tables, checks, grid=1, K=1, duration_ms=0, table_bytes=None, n_checks=None,
                      zap=-1):
        cap = max(grid, 1)
        recs = (CtRecord * cap)()
        n, ms = C.c_int(), C.c_float()
        tables = np.ascontiguousarray(tables, dtype=np.uint32)
        checks = np.ascontiguousarray(checks, dtype=np.uint32)
        rc = self.L.l1k_run_tables(self.h, fmt, seed, tables.ctypes.data,
                                   tables.nbytes if table_bytes is None else table_bytes, checks.ctypes.data,
                                   checks.size if n_checks is None else n_checks, grid, K, int(duration_ms * MS), zap,
                                   recs, cap, C.byref(n), C.byref(ms))
        return rc, list(recs[:n.value]) if rc == 0 else []


@pytest.fixture(scope="module")
def H():
    if not os.path.exists(LIB_PATH):
        pytest.skip("run __graft_entry__.build() first")
    h = Harness(0)
    yield h
    h.close()


def _complete(r):
    return r.rounds >= 1 and r.comparisons == r.rounds * TILES * REPS


def _gpu_busy():
    """True if NVML lists a compute process on GPU 0 besides this one (the rule b2dp_l1_test applies)."""
    try:
        import pynvml
        pynvml.nvmlInit()
        return len(pynvml.nvmlDeviceGetComputeRunningProcesses(pynvml.nvmlDeviceGetHandleByIndex(0))) > 1
    except Exception:       # noqa: BLE001
        return None


@pytest.mark.parametrize("fmt", FORMATS, ids=FMT_IDS)
@pytest.mark.parametrize("seed", [1, 0xC0FFEE])
def test_dump_equals_reference(H, ref, fmt, seed):
    recs, _, K, got = H.run(fmt, seed, 0, dump=True)
    if fmt == lo.DATA:
        want = np.stack([ref.span(seed, t, K) for t in range(TILES)])
    else:
        want = ref.launch_tables(seed, fmt)[1]
    got = got.reshape(want.shape)
    bad = np.argwhere(got != want)
    where = ""
    if bad.size and fmt == lo.TEX:
        where = " (op %s)" % sorted({TEX_OPS[(int(b[2]) % 32) // 4] for b in bad})
    assert bad.size == 0, "first differing (tile, thread, word): %s got %#x want %#x (%d words differ)%s" % (
        tuple(bad[0]), got[tuple(bad[0])], want[tuple(bad[0])], len(bad), where)
    assert len(recs) == 1 and recs[0].mismatches == 0 and _complete(recs[0])


@pytest.mark.parametrize("fmt", FORMATS, ids=FMT_IDS)
def test_clean_runs_cover_every_sm(H, fmt):
    occ = H.occupancy(fmt)
    for i, seed in enumerate((0x5EED0000, 0x5EED0001, 0x5EED0002)):
        recs, _, _, _ = H.run(fmt, seed, 100 if i == 0 else 0)
        assert len(recs) == H.sms * occ
        for r in recs:
            assert _complete(r) and r.mismatches == 0, (seed, r.smid, r.rounds, r.comparisons, r.mismatches)
        per_sm = {}
        for r in recs:
            per_sm[r.smid] = per_sm.get(r.smid, 0) + 1
        assert len(per_sm) == H.sms, sorted(per_sm)
        if not _gpu_busy():
            assert set(per_sm.values()) == {occ}, per_sm


@pytest.mark.parametrize("fmt", FORMATS, ids=FMT_IDS)
def test_wrong_check_counted_in_its_tile(H, ref, fmt):
    tables, _, checks = ref.launch_tables(7, fmt)
    for t in (0, 37, 127):
        tile = t % TILES
        c = checks.copy()
        c[tile, t] ^= np.uint32(1 << (t % 32))
        rc, recs = H.run_tables_rc(fmt, 7, tables, c, grid=2)
        assert rc == 0 and len(recs) == 2
        for r in recs:
            assert r.rounds == 1 and r.comparisons == TILES * REPS
            assert r.mismatches == REPS and r.first_bad_tile == tile and r.first_bad_rep == 0, (t, r.mismatches)


@pytest.mark.parametrize("fmt", FORMATS, ids=FMT_IDS)
def test_malformed_tables_and_handles_refused(H, ref, fmt):
    tables, _, checks = ref.launch_tables(3, fmt)
    assert H.run_tables_rc(fmt, 3, tables, checks, table_bytes=tables.nbytes - 4)[0] not in (0, 1)
    assert H.run_tables_rc(fmt, 3, tables, checks, n_checks=checks.size - 1)[0] not in (0, 1)
    assert H.run_tables_rc(fmt, 3, tables, checks, grid=0)[0] not in (0, 1)
    bad = tables.copy()
    if fmt == lo.DATA:
        bad[4 * 5] = 5                    # no such background
    elif fmt == lo.TEX:
        bad[4 * 5] &= ~np.uint32(1)       # an even multiplier is no permutation
    else:
        bad[4 * 5] = 4                    # no such window
    assert H.run_tables_rc(fmt, 3, bad, checks)[0] == -3
    if fmt == lo.TEX:
        for z in (0, 4):
            assert H.run_tables_rc(fmt, 3, tables, checks, zap=z)[0] == -6


def _fault_cases():
    out = []
    for fmt in FORMATS:
        for f in lo.FAULTS[fmt]:
            if fmt == lo.DATA and f[0].startswith("stuck") and f[3] not in (0, 31):
                continue
            out.append((fmt, f))
    return out


@pytest.mark.parametrize("fmt,fault", _fault_cases())
def test_fault_model_checks_mismatch_where_the_model_says(H, fmt, fault):
    """Check values a device with the fault would match: this healthy H100 mismatches them in every repetition of every
    tile where the model changes the check, and nowhere else (the tables are the oracle's, which equal the C++)."""
    seed = 0xFA17
    tables = np.array([lo.table(seed, fmt, t) for t in range(TILES)], dtype=np.uint64).astype(np.uint32).ravel()
    if fmt == lo.DATA:   # the even fold is the check; the kernel derives the odd repetitions' from it
        bad = np.array([[e for e, _ in lo.checks(seed, fmt, t, fault=fault)] for t in range(TILES)], dtype=np.uint64)
        clean = np.array([[e for e, _ in lo.checks(seed, fmt, t)] for t in range(TILES)], dtype=np.uint64)
    else:
        bad = np.array([lo.checks(seed, fmt, t, fault=fault) for t in range(TILES)], dtype=np.uint64)
        clean = np.array([lo.checks(seed, fmt, t) for t in range(TILES)], dtype=np.uint64)
    tiles = [t for t in range(TILES) if (bad[t] != clean[t]).any()]
    if fmt != lo.DATA:
        assert tiles == list(range(TILES)), fault
    rc, recs = H.run_tables_rc(fmt, seed, tables, bad.astype(np.uint32), grid=1)
    assert rc == 0 and len(recs) == 1
    r = recs[0]
    assert r.rounds == 1 and r.comparisons == TILES * REPS
    assert r.mismatches == REPS * len(tiles), (fault, r.mismatches, tiles)
    if tiles:
        assert (r.first_bad_tile, r.first_bad_rep) == (tiles[0], 0)
    rc, recs = H.run_tables_rc(fmt, seed, tables, clean.astype(np.uint32), grid=1)
    assert rc == 0 and recs[0].mismatches == 0


# ---- through the ABI ---------------------------------------------------------------------------------------------------
@pytest.fixture(scope="module")
def pkg():
    sys.path.insert(0, ROOT)
    import importlib
    return importlib.import_module("k8s-device-plugin_b200")


def _open(pkg, nbytes=64 * MiB):
    return pkg.Context("cuda:devices=0,bytes=%d,calib=1" % nbytes)


@pytest.fixture(scope="module")
def sm_ids(H):
    recs, _, _, _ = H.run(lo.CONST, 0x5EED, 20)
    assert all(_complete(r) and r.mismatches == 0 for r in recs)
    return sorted({r.smid for r in recs})


def test_l1_test_clean_and_memory_back(pkg):
    import torch
    torch.cuda.init()
    N = pkg._native
    with _open(pkg) as ctx:
        ctx.l1_test(0, duration_ms=10)                          # first launch loads the kernels: not counted below
        free0, _ = torch.cuda.mem_get_info(0)
        (r,) = ctx.l1_test(0, duration_ms=100)
        free1, _ = torch.cuda.mem_get_info(0)
        assert r.healthy and r.err == 0, r
        assert r.mismatches == [0, 0, 0] and r.bad_sm_mask == [0, 0, 0, 0], r
        assert (r.first_bad_sm, r.first_bad_format, r.first_bad_tile) == (-1, -1, -1)
        assert r.sm_count == torch.cuda.get_device_properties(0).multi_processor_count
        assert all(ms >= 90 for ms in r.ms) and all(t > 0 for t in r.tflops), r
        if not _gpu_busy():
            assert r.sms_covered == r.sm_count and not r.flags & ~(N.CT_NO_ECC | N.CT_ECC_CORRECTED), r
        assert abs(free1 - free0) < 2 * MiB, (free0, free1)
        (p,) = ctx.probe_health(min_gbs=1e-3)
        assert p.healthy and not p.flags & N.RES_COMPUTE


@pytest.mark.parametrize("where,mask", [("first", 0x1), ("middle", 0x80000000), ("last", 0xFFFFFFFF)])
def test_l1_test_fault_is_attributed_and_latched_until_reset(pkg, H, sm_ids, where, mask):
    N = pkg._native
    s = {"first": sm_ids[0], "middle": sm_ids[len(sm_ids) // 2], "last": sm_ids[-1]}[where]
    with _open(pkg) as ctx:
        (r,) = ctx.l1_test(0, duration_ms=10, fault_sm=s, fault_mask=mask)
        assert not r.healthy and r.err == 0, r
        assert r.bad_sms() == [s], r.bad_sms()
        assert (r.first_bad_sm, r.first_bad_format, r.first_bad_tile) == (s, N.L1_DATA, 0), r
        for f in FORMATS:          # one mismatch per CTA that ran on s
            assert 1 <= r.mismatches[f] <= H.occupancy(f), (f, r.mismatches)
        (p,) = ctx.probe_health(min_gbs=1e-3)
        assert p.flags & N.RES_COMPUTE and not p.healthy and p.mismatches == 0
        ctx.probe_reset(0)
        (p,) = ctx.probe_health(min_gbs=1e-3)
        assert p.healthy and not p.flags & N.RES_COMPUTE


def test_l1_test_two_contexts_at_once_stay_healthy(pkg):
    """Two contexts in one process share the device's constant bank; each call loads it with its own seed.  Run at
    once from two threads, neither may read the other's bank."""
    import threading
    out, errs = {}, []

    def one(k):
        try:
            with _open(pkg) as ctx:
                out[k] = [ctx.l1_test(0, duration_ms=100)[0] for _ in range(3)]
        except Exception as e:       # noqa: BLE001
            errs.append(e)
    ts = [threading.Thread(target=one, args=(k,)) for k in range(2)]
    for t in ts:
        t.start()
    for t in ts:
        t.join()
    assert not errs, errs
    for k in range(2):
        for r in out[k]:
            assert r.healthy and r.err == 0 and r.mismatches == [0, 0, 0], (k, r)
    assert len({r.seed for k in range(2) for r in out[k]}) > 1


def test_l1_test_skips_a_busy_gpu(pkg):
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
            (r,) = ctx.l1_test(0, duration_ms=10, fault_sm=0, fault_mask=1)
            assert r.flags & N.CT_SKIPPED_BUSY and r.mismatches == [0, 0, 0] and r.ms == [0, 0, 0], r
            (p,) = ctx.probe_health(min_gbs=1e-3)
            assert not p.flags & N.RES_COMPUTE
            (r,) = ctx.l1_test(0, duration_ms=10, even_if_busy=True)
            assert not r.flags & N.CT_SKIPPED_BUSY and r.healthy and r.err == 0, r
    finally:
        if helper.poll() is None:
            helper.kill()
        helper.wait()


def test_daemon_l1_test_at_start(tmp_path):
    exe = os.path.join(ROOT, "k8s-device-plugin_b200", "b200dp_plugind")
    if not os.path.exists(exe):
        pytest.skip("no daemon build")
    d = tmp_path / "p"
    d.mkdir()
    proc = subprocess.Popen([exe, "-backend=cuda:devices=0,bytes=67108864,calib=1", "-plugin_dir", str(d),
                             "-start_retry_wait=0.05", "-l1_test_at_start=1", "-compute_test_ms=50"],
                            stderr=subprocess.PIPE, text=True)
    line = ""
    try:
        for _ in range(200):
            line = proc.stderr.readline()
            if ("L1 test" in line and ("ealthy" in line or "not run" in line)) or not line:
                break
    finally:
        proc.terminate()
        try:
            proc.wait(timeout=10)
        except subprocess.TimeoutExpired:
            proc.kill()
            proc.wait()
    assert "L1 test" in line and "Healthy" in line and "Unhealthy" not in line, line
