"""The on-demand FP32 / FP64 self-test on a real H100.

- The kernel of fp_selftest.cuh, launched directly (tests/native/libfp_test_kernels_test.so):
  - the DUMP instantiation's result words equal tests/fp_test_oracle.py bit for bit, for every format and tile at two
    seeds.  This is the measurement that the H100's FFMA and DFMA are fused, round to nearest-even and keep
    subnormals, and that DMMA is exact below 2^53 with the fragment layout fp_test_math.hpp assumes;
  - a clean run covers every SM id and every CTA compares exactly what its rounds hold;
  - on caller-built tables: a wrong check value in any of the 128 threads is counted in exactly its tile's 16
    repetitions; a wrong x, a or b (A or B for DMMA) in every repetition of every round by every CTA; and check values
    built by a unit that rounds ties away from zero, flushes subnormal results or rounds the product before the add
    mismatch in every tile;
  - malformed tables are refused before anything runs.
- b2dp_fp_test through the ABI: Healthy on an idle card, memory handed back, the probe ring untouched, the fault hook
  attributed to its SM and latched until probe_reset, the busy skip, and the daemon's -fp_test_at_start.

Every run is short: 10-100 ms per format."""
import ctypes as C
import os
import signal
import subprocess
import sys
import time

import numpy as np
import pytest

import fp_test_oracle as ft
from oracle import probe as oprobe

pytestmark = pytest.mark.gpu

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(HERE)
LIB_PATH = os.path.join(HERE, "native", "libfp_test_kernels_test.so")
MiB = 1 << 20
MS = 1000000
FMT_IDS = [ft.NAMES[f] for f in ft.FORMATS]


class CtRecord(C.Structure):
    _fields_ = [("smid", C.c_uint32), ("nsmid", C.c_uint32), ("rounds", C.c_uint64), ("comparisons", C.c_uint64),
                ("mismatches", C.c_uint64), ("first_bad_tile", C.c_int32), ("first_bad_rep", C.c_int32),
                ("seq", C.c_uint64)]


_P = C.POINTER


class Harness:
    def __init__(self, device=0):
        L = C.CDLL(LIB_PATH)
        L.fk_open.restype = C.c_void_p
        L.fk_open.argtypes = [C.c_int, C.c_char_p, C.c_int]
        L.fk_close.argtypes = [C.c_void_p]
        L.fk_error.restype = C.c_char_p
        L.fk_error.argtypes = [C.c_void_p]
        L.fk_sms.argtypes = [C.c_void_p]
        L.fk_table_bytes.restype = C.c_uint64
        L.fk_occupancy.argtypes = [C.c_void_p, C.c_int, _P(C.c_int)]
        L.fk_dump.argtypes = [C.c_void_p, C.c_int, C.c_uint32, _P(C.c_uint32), _P(CtRecord)]
        L.fk_run.argtypes = [C.c_void_p, C.c_int, C.c_uint32, C.c_uint64, C.c_int, C.c_uint32, _P(CtRecord), C.c_int,
                             _P(C.c_int), _P(C.c_float)]
        L.fk_run_tables.argtypes = [C.c_void_p, C.c_int, C.c_int, C.c_void_p, C.c_uint64, C.c_void_p, C.c_uint64,
                                    C.c_int, C.c_uint64, _P(CtRecord), C.c_int, _P(C.c_int), _P(C.c_float),
                                    _P(C.c_uint32)]
        assert L.fk_record_bytes() == C.sizeof(CtRecord)
        assert (L.fk_tiles(), L.fk_reps()) == (ft.TILES, ft.REPS)
        assert [L.fk_words(f) for f in ft.FORMATS] == [ft.WORDS[f] for f in ft.FORMATS]
        self.L = L
        err = C.create_string_buffer(512)
        self.h = L.fk_open(device, err, len(err))
        if not self.h:
            raise RuntimeError("fk_open: " + err.value.decode())
        self.sms = L.fk_sms(self.h)

    def close(self):
        if self.h:
            self.L.fk_close(self.h)
            self.h = None

    def _check(self, rc, what):
        if rc == 1:
            raise RuntimeError("%s: %s" % (what, self.L.fk_error(self.h).decode()))
        assert rc == 0, "%s refused: code %d" % (what, rc)

    def occupancy(self, fmt):
        n = C.c_int()
        self._check(self.L.fk_occupancy(self.h, fmt, C.byref(n)), "fk_occupancy")
        return n.value

    def dump(self, fmt, seed):
        out = np.zeros(ft.TILES * ft.THREADS * ft.WORDS[fmt], dtype=np.uint32)
        rec = CtRecord()
        self._check(self.L.fk_dump(self.h, fmt, seed, out.ctypes.data_as(_P(C.c_uint32)), C.byref(rec)), "fk_dump")
        return out.reshape(ft.TILES, ft.THREADS, ft.WORDS[fmt]), rec

    def run(self, fmt, seed, duration_ms, fault_sm=-1, fault_mask=0):
        cap = self.sms * 32
        recs = (CtRecord * cap)()
        n, ms = C.c_int(), C.c_float()
        self._check(self.L.fk_run(self.h, fmt, seed, int(duration_ms * MS), fault_sm, fault_mask, recs, cap,
                                  C.byref(n), C.byref(ms)), "fk_run")
        return list(recs[:n.value]), ms.value

    def run_tables_rc(self, fmt, tables, checks, grid=1, duration_ms=0, dump=False, table_bytes=None, n_checks=None):
        cap = max(grid, 1)
        recs = (CtRecord * cap)()
        n, ms = C.c_int(), C.c_float()
        out = np.zeros(ft.TILES * ft.THREADS * ft.WORDS[fmt], dtype=np.uint32) if dump else None
        rc = self.L.fk_run_tables(self.h, fmt, int(dump), tables.ctypes.data, tables.nbytes if table_bytes is None
                                  else table_bytes, checks.ctypes.data, checks.size if n_checks is None else n_checks,
                                  grid, int(duration_ms * MS), recs, cap, C.byref(n), C.byref(ms),
                                  out.ctypes.data_as(_P(C.c_uint32)) if dump else None)
        return rc, list(recs[:n.value]) if rc == 0 else [], out

    def run_tables(self, fmt, tables, checks, grid=1, duration_ms=0):
        rc, recs, _ = self.run_tables_rc(fmt, tables, checks, grid, duration_ms)
        self._check(rc, "fk_run_tables")
        return recs


@pytest.fixture(scope="module")
def H():
    if not os.path.exists(LIB_PATH):
        pytest.skip("run __graft_entry__.build() first")
    h = Harness(0)
    yield h
    h.close()


def _gpu_busy():
    """True if NVML lists a compute process on GPU 0 besides this one (the rule b2dp_fp_test applies)."""
    try:
        import pynvml
        pynvml.nvmlInit()
        return len(pynvml.nvmlDeviceGetComputeRunningProcesses(pynvml.nvmlDeviceGetHandleByIndex(0))) > 1
    except Exception:       # noqa: BLE001
        return None


# ---- tables from the oracle -------------------------------------------------------------------------------------------------
_TILES = {}


def oracle_tiles(seed, fmt):
    """[tile] -> (table, words, checks, operands), cached."""
    if (seed, fmt) not in _TILES:
        _TILES[seed, fmt] = [ft.tile(seed, fmt, t) for t in range(ft.TILES)]
    return _TILES[seed, fmt]


def launch_tables(seed, fmt):
    """The launch inputs: tables (TILES x SLOTS x THREADS values) and checks (TILES x THREADS), as numpy arrays."""
    tiles = oracle_tiles(seed, fmt)
    dt = np.uint32 if fmt == ft.FP32 else np.uint64
    tables = np.array([t[0] for t in tiles], dtype=dt)
    checks = np.array([t[2] for t in tiles], dtype=np.uint32)
    return tables, checks


# ---- the kernel, directly ---------------------------------------------------------------------------------------------
@pytest.mark.parametrize("seed", [0x0, 0xC0FFEE17])
@pytest.mark.parametrize("fmt", ft.FORMATS, ids=FMT_IDS)
def test_dump_matches_the_oracle_bit_for_bit(H, fmt, seed):
    got, rec = H.dump(fmt, seed)
    bad = []
    for t, (_, words, _, _) in enumerate(oracle_tiles(seed, fmt)):
        want = np.array(words, dtype=np.uint32)
        if not np.array_equal(got[t], want):
            idx = np.argwhere(got[t] != want)
            th, j = idx[0]
            bad.append("tile %d: %d of %d words differ; first thread %d word %d got 0x%08x want 0x%08x"
                       % (t, len(idx), want.size, th, j, got[t][th, j], want[th, j]))
    assert not bad, "\n".join(bad)
    assert (rec.seq, rec.rounds, rec.comparisons, rec.mismatches) == (7, 1, ft.TILES * ft.REPS, 0), \
        (rec.seq, rec.rounds, rec.comparisons, rec.mismatches)
    assert (rec.first_bad_tile, rec.first_bad_rep) == (-1, -1)


def _check_clean(recs, seq=7):
    for r in recs:
        assert r.seq == seq and r.rounds >= 1 and r.comparisons == r.rounds * ft.TILES * ft.REPS, \
            (r.smid, r.seq, r.rounds, r.comparisons)
        assert r.mismatches == 0 and (r.first_bad_tile, r.first_bad_rep) == (-1, -1)
        assert r.smid < r.nsmid <= 256


@pytest.fixture(scope="module")
def sm_ids(H):
    recs, _ = H.run(ft.FP32, 0x5EED, 20)
    _check_clean(recs)
    return sorted({r.smid for r in recs})


MACS = {ft.FP32: ft.THREADS * ft.RESULTS, ft.FP64: ft.THREADS * ft.RESULTS, ft.DMMA: 4 * 16 * 16 * 8 * 16}


@pytest.mark.parametrize("fmt", ft.FORMATS, ids=FMT_IDS)
def test_clean_run_covers_every_sm(H, fmt):
    duration = 100
    recs, ms = H.run(fmt, 0x1234567 + fmt, duration)
    assert len(recs) == H.sms * H.occupancy(fmt)
    _check_clean(recs)
    assert ms >= duration * 0.9
    flops = 2 * MACS[fmt] * sum(r.comparisons for r in recs)
    print("%s: %d CTAs (%d resident per SM), %d SM ids, %.1f ms, %.1f TFLOP/s"
          % (ft.NAMES[fmt], len(recs), H.occupancy(fmt), len({r.smid for r in recs}), ms, flops / ms * 1e-9))
    if _gpu_busy():
        pytest.skip("another process uses the GPU: coverage is not asserted (the rest was)")
    assert len({r.smid for r in recs}) == H.sms


@pytest.mark.parametrize("fmt", ft.FORMATS, ids=FMT_IDS)
def test_wrong_check_value_in_every_thread_is_counted_in_its_tile(H, fmt):
    tables, checks = launch_tables(0xC4EC, fmt)
    for t in range(ft.THREADS):
        tile = t % ft.TILES
        bad = checks.copy()
        bad[tile, t] ^= np.uint32(1 << (t % 32))
        (r,) = H.run_tables(fmt, tables, bad)
        assert (r.seq, r.rounds, r.comparisons) == (7, 1, ft.TILES * ft.REPS)
        assert (r.mismatches, r.first_bad_tile, r.first_bad_rep) == (ft.REPS, tile, 0), (t, r.mismatches, r.first_bad_tile)


def _corrupt_operand(seed, fmt, tile, thread, slot, bit):
    """Tables with one operand bit flipped, the oracle's check of that thread with it, and the clean tables."""
    tables, checks = launch_tables(seed, fmt)
    bad = tables.copy()
    bad[tile, slot, thread] ^= bad.dtype.type(1 << bit)
    if fmt != ft.DMMA:
        x, a, b = (list(v) for v in oracle_tiles(seed, fmt)[tile][3][thread])
        ops = x + a + b
        ops[slot] = int(bad[tile, slot, thread])
        words = ft.fma_words(fmt, ops[:ft.NX], ops[ft.NX:ft.NX + ft.NAB], ops[ft.NX + ft.NAB:])
        assert ft.fold(words) != checks[tile, thread], "the flip must change the thread's results"
    return bad, checks


OPERAND_CASES = [  # (fmt, tile, thread, slot, bit): x, a and b of FP32 / FP64, A and B of DMMA, in several warps
    (ft.FP32, 0, 0, 3, 5), (ft.FP32, 3, 77, 8 + 6, 22), (ft.FP32, 7, 127, 24 + 15, 30),
    (ft.FP64, 1, 33, 0, 51), (ft.FP64, 4, 64, 8 + 2, 0), (ft.FP64, 6, 100, 24 + 9, 63),
    (ft.DMMA, 2, 5, 3, 40), (ft.DMMA, 5, 96, 32 + 2, 20), (ft.DMMA, 7, 127, 47, 52),
]


@pytest.mark.parametrize("fmt,tile,thread,slot,bit", OPERAND_CASES)
def test_wrong_operand_is_counted_in_every_repetition_of_every_round_by_every_cta(H, fmt, tile, thread, slot, bit):
    tables, checks = _corrupt_operand(0x0BAD, fmt, tile, thread, slot, bit)
    grid = H.sms * H.occupancy(fmt)
    recs = H.run_tables(fmt, tables, checks, grid=grid, duration_ms=10)
    assert len(recs) == grid
    for r in recs:
        assert r.seq == 7 and r.comparisons == r.rounds * ft.TILES * ft.REPS
        assert (r.mismatches, r.first_bad_tile, r.first_bad_rep) == (r.rounds * ft.REPS, tile, 0), \
            (r.smid, r.rounds, r.mismatches, r.first_bad_tile)


@pytest.mark.parametrize("rule", ["ties_away", "ftz", "unfused"])
@pytest.mark.parametrize("fmt", [ft.FP32, ft.FP64], ids=FMT_IDS[:2])
def test_checks_of_a_non_ieee_unit_mismatch_in_every_tile(H, fmt, rule):
    """Every tile holds ties, subnormal results and cancellations, so a unit that breaks any of these rules would
    disagree with the host in every tile: the kernel counts all of them."""
    seed = 0x1EEE
    tables, checks = launch_tables(seed, fmt)
    wrong = checks.copy()
    for t, (_, _, _, ops) in enumerate(oracle_tiles(seed, fmt)):
        for th, (x, a, b) in enumerate(ops):
            wrong[t, th] = ft.fold(ft.fma_words(fmt, x, a, b, rule))
    assert all((wrong[t] != checks[t]).any() for t in range(ft.TILES))
    recs = H.run_tables(fmt, tables, wrong, grid=4)
    for r in recs:
        assert (r.rounds, r.mismatches, r.first_bad_tile, r.first_bad_rep) == (1, ft.TILES * ft.REPS, 0, 0), \
            (r.rounds, r.mismatches)
    # and the correct checks pass on the same tables
    _check_clean(H.run_tables(fmt, tables, checks, grid=4))


def test_run_tables_refuses_malformed_input(H):
    tables, checks = launch_tables(0, ft.FP32)
    assert H.run_tables_rc(3, tables, checks)[0] == -1
    assert H.run_tables_rc(ft.FP32, tables, checks, table_bytes=tables.nbytes - 4)[0] == -3
    assert H.run_tables_rc(ft.FP64, tables, checks)[0] == -3          # an FP32 table is half an FP64 one
    assert H.run_tables_rc(ft.FP32, tables, checks, n_checks=checks.size - 1)[0] == -3
    assert H.run_tables_rc(ft.FP32, tables, checks, grid=0)[0] == -4
    assert H.run_tables_rc(ft.FP32, tables, checks, grid=H.sms * 64)[0] == -4


# ---- through the ABI --------------------------------------------------------------------------------------------------
def _open(pkg, nbytes=64 * MiB):
    return pkg.Context("cuda:devices=0,bytes=%d,calib=1" % nbytes)


def test_fp_test_clean_memory_back_and_ring_untouched(pkg):
    import torch
    torch.cuda.init()
    N = pkg._native
    nbytes = 64 * MiB
    n_words = nbytes // 4
    with _open(pkg, nbytes) as ctx:
        ctx.fp_test(0, duration_ms=10)                         # first launch loads the kernels: not counted below
        (p0,) = ctx.probe_health(min_gbs=1e-3)
        seed = oprobe.next_seed(p0.seed)
        src = ctx.probe_peek(0, 0, n_words)
        free0, _ = torch.cuda.mem_get_info(0)
        (r,) = ctx.fp_test(0, duration_ms=100)
        free1, _ = torch.cuda.mem_get_info(0)
        assert r.healthy and r.err == 0, r
        assert r.mismatches == [0, 0, 0] and r.bad_sm_mask == [0, 0, 0, 0], r
        assert (r.first_bad_sm, r.first_bad_format, r.first_bad_tile) == (-1, -1, -1)
        assert r.sm_count == torch.cuda.get_device_properties(0).multi_processor_count
        assert r.nsmid >= r.sm_count and all(ms >= 90 for ms in r.ms) and all(t > 0 for t in r.tflops), r
        if not _gpu_busy():
            assert r.sms_covered == r.sm_count and not r.flags & N.CT_PARTIAL_COVERAGE, r
        assert abs(free1 - free0) < 2 * MiB, (free0, free1)
        assert np.array_equal(ctx.probe_peek(0, 0, n_words), src)
        (p,) = ctx.probe_health(min_gbs=1e-3)
        cs, bad, first, _ = oprobe.probe_pass(src, seed, oprobe.next_seed(seed))
        assert (p.seed, p.checksum, p.mismatches) == (seed, cs, bad) and p.healthy
        assert not p.flags & N.RES_COMPUTE
    print("fp test 100 ms/format: SMs %d/%d, ms %s, TFLOP/s fp32 %.1f fp64 %.1f dmma %.1f"
          % (r.sms_covered, r.sm_count, ["%.1f" % x for x in r.ms], *r.tflops))


@pytest.mark.parametrize("where,mask", [("first", 0x1), ("middle", 0x80000000), ("last", 0x1)])
def test_fp_test_fault_is_attributed_and_latched_until_reset(pkg, H, sm_ids, where, mask):
    N = pkg._native
    s = {"first": sm_ids[0], "middle": sm_ids[len(sm_ids) // 2], "last": sm_ids[-1]}[where]
    with _open(pkg) as ctx:
        (r,) = ctx.fp_test(0, duration_ms=10, fault_sm=s, fault_mask=mask)
        assert not r.healthy and r.err == 0, r
        assert r.bad_sms() == [s], r.bad_sms()
        assert (r.first_bad_sm, r.first_bad_format, r.first_bad_tile) == (s, N.FT_FP32, 0), r
        for f in ft.FORMATS:          # one mismatch per CTA that ran on s
            assert 1 <= r.mismatches[f] <= H.occupancy(f), (f, r.mismatches)
        (p,) = ctx.probe_health(min_gbs=1e-3)
        assert p.flags & N.RES_COMPUTE and not p.healthy and p.mismatches == 0
        _, st = ctx.list_and_watch("gpu", N.LW_HEARTBEAT, min_gbs=1e-3)
        assert st.n_unhealthy == 1
        ctx.probe_reset(0)
        (p,) = ctx.probe_health(min_gbs=1e-3)
        assert p.healthy and not p.flags & N.RES_COMPUTE


def test_fp_test_skips_a_busy_gpu(pkg):
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
            (r,) = ctx.fp_test(0, duration_ms=10, fault_sm=0, fault_mask=1)
            assert r.flags & N.CT_SKIPPED_BUSY and r.mismatches == [0, 0, 0] and r.ms == [0, 0, 0], r
            (p,) = ctx.probe_health(min_gbs=1e-3)
            assert not p.flags & N.RES_COMPUTE
            (r,) = ctx.fp_test(0, duration_ms=10, even_if_busy=True)
            assert not r.flags & N.CT_SKIPPED_BUSY and r.healthy and r.err == 0, r
    finally:
        if helper.poll() is None:
            helper.kill()
        helper.wait()


def _daemon_lines(short_dir, level):
    exe = os.path.join(ROOT, "k8s-device-plugin_b200", "b200dp_plugind")
    proc = subprocess.Popen([exe, "-backend=cuda:devices=0,bytes=67108864,calib=1", "-plugin_dir", short_dir,
                             "-start_retry_wait=0.05", "-fp_test_at_start=%d" % level, "-compute_test_ms=50"],
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
    assert log.index("fp test ") < log.index("Failed to start plugin"), log[-3000:]  # before the first registration
    return [ln for ln in log.splitlines() if ln.startswith("fp test ")], log


def test_daemon_fp_test_at_start_logs_a_clean_result(short_dir):
    lines, log = _daemon_lines(short_dir, 1)
    assert len(lines) == 1, log[-3000:]
    if "flags 0x1," in lines[0]:
        lines, log = _daemon_lines(short_dir, 2)
        assert len(lines) == 1, log[-3000:]
    assert ": Healthy, flags 0x" in lines[0] and "mismatches 0/0/0, first bad SM -1" in lines[0], log[-3000:]
