"""The on-demand integer and warp-exchange self-test on a real H100.

- The kernel of int_selftest.cuh, launched directly (tests/native/libint_test_kernels_test.so):
  - the DUMP instantiation's result words equal tests/int_test_oracle.py word for word, for every format and tile at two
    seeds: this H100's integer pipes and shuffle network agree with the PTX ISA on every crafted class;
  - a clean run covers every SM id and every CTA compares exactly what its rounds hold, at 32 seeds per format through
    the product's table builder;
  - on caller-built tables: a wrong check value in any of the 128 threads is counted in exactly its tile's 16
    repetitions; a changed operand word in every repetition of every round by every CTA; and check values computed by
    a fault model of tests/test_int_test_cpu.py mismatch in the tiles the model says;
  - malformed tables are refused before anything runs.
- b2dp_int_test through the ABI: Healthy on an idle card, the fault hook attributed to its SM and latched until
  probe_reset, the busy skip, and the daemon's -int_test_at_start.

Every run is short: 0-100 ms per format."""
import ctypes as C
import os
import signal
import subprocess
import sys
import time

import numpy as np
import pytest

import int_test_oracle as it

pytestmark = pytest.mark.gpu

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(HERE)
LIB_PATH = os.path.join(HERE, "native", "libint_test_kernels_test.so")
MiB = 1 << 20
MS = 1000000
FORMATS = (it.MAD, it.BIT, it.WARP)
FMT_IDS = ["mad", "bit", "warp"]


class CtRecord(C.Structure):
    _fields_ = [("smid", C.c_uint32), ("nsmid", C.c_uint32), ("rounds", C.c_uint64), ("comparisons", C.c_uint64),
                ("mismatches", C.c_uint64), ("first_bad_tile", C.c_int32), ("first_bad_rep", C.c_int32),
                ("seq", C.c_uint64)]


_P = C.POINTER


class Harness:
    def __init__(self, device=0):
        L = C.CDLL(LIB_PATH)
        L.ik_open.restype = C.c_void_p
        L.ik_open.argtypes = [C.c_int, C.c_char_p, C.c_int]
        L.ik_close.argtypes = [C.c_void_p]
        L.ik_error.restype = C.c_char_p
        L.ik_error.argtypes = [C.c_void_p]
        L.ik_sms.argtypes = [C.c_void_p]
        L.ik_table_bytes.restype = C.c_uint64
        L.ik_occupancy.argtypes = [C.c_void_p, C.c_int, _P(C.c_int)]
        L.ik_dump.argtypes = [C.c_void_p, C.c_int, C.c_uint32, _P(C.c_uint32), _P(CtRecord)]
        L.ik_run.argtypes = [C.c_void_p, C.c_int, C.c_uint32, C.c_uint64, C.c_int, C.c_uint32, _P(CtRecord), C.c_int,
                             _P(C.c_int), _P(C.c_float)]
        L.ik_run_tables.argtypes = [C.c_void_p, C.c_int, C.c_int, C.c_void_p, C.c_uint64, C.c_void_p, C.c_uint64,
                                    C.c_int, C.c_uint64, _P(CtRecord), C.c_int, _P(C.c_int), _P(C.c_float),
                                    _P(C.c_uint32)]
        assert L.ik_record_bytes() == C.sizeof(CtRecord)
        assert (L.ik_tiles(), L.ik_reps()) == (it.TILES, it.REPS)
        assert [L.ik_words(f) for f in FORMATS] == list(it.WORDS)
        assert [L.ik_table_bytes(f) for f in FORMATS] == [4 * it.THREADS * s for s in it.SLOTS]
        self.L = L
        err = C.create_string_buffer(512)
        self.h = L.ik_open(device, err, len(err))
        if not self.h:
            raise RuntimeError("ik_open: " + err.value.decode())
        self.sms = L.ik_sms(self.h)

    def close(self):
        if self.h:
            self.L.ik_close(self.h)
            self.h = None

    def _check(self, rc, what):
        if rc == 1:
            raise RuntimeError("%s: %s" % (what, self.L.ik_error(self.h).decode()))
        assert rc == 0, "%s refused: code %d" % (what, rc)

    def occupancy(self, fmt):
        n = C.c_int()
        self._check(self.L.ik_occupancy(self.h, fmt, C.byref(n)), "ik_occupancy")
        return n.value

    def dump(self, fmt, seed):
        out = np.zeros(it.TILES * it.THREADS * it.WORDS[fmt], dtype=np.uint32)
        rec = CtRecord()
        self._check(self.L.ik_dump(self.h, fmt, seed, out.ctypes.data_as(_P(C.c_uint32)), C.byref(rec)), "ik_dump")
        return out.reshape(it.TILES, it.THREADS, it.WORDS[fmt]), rec

    def run(self, fmt, seed, duration_ms, fault_sm=-1, fault_mask=0):
        cap = self.sms * 32
        recs = (CtRecord * cap)()
        n, ms = C.c_int(), C.c_float()
        self._check(self.L.ik_run(self.h, fmt, seed, int(duration_ms * MS), fault_sm, fault_mask, recs, cap,
                                  C.byref(n), C.byref(ms)), "ik_run")
        return list(recs[:n.value]), ms.value

    def run_tables_rc(self, fmt, tables, checks, grid=1, duration_ms=0, table_bytes=None, n_checks=None):
        cap = max(grid, 1)
        recs = (CtRecord * cap)()
        n, ms = C.c_int(), C.c_float()
        rc = self.L.ik_run_tables(self.h, fmt, 0, tables.ctypes.data, tables.nbytes if table_bytes is None
                                  else table_bytes, checks.ctypes.data, checks.size if n_checks is None else n_checks,
                                  grid, int(duration_ms * MS), recs, cap, C.byref(n), C.byref(ms), None)
        return rc, list(recs[:n.value]) if rc == 0 else []

    def run_tables(self, fmt, tables, checks, grid=1, duration_ms=0):
        rc, recs = self.run_tables_rc(fmt, tables, checks, grid, duration_ms)
        self._check(rc, "ik_run_tables")
        return recs


@pytest.fixture(scope="module")
def H():
    if not os.path.exists(LIB_PATH):
        pytest.skip("run __graft_entry__.build() first")
    h = Harness(0)
    yield h
    h.close()


def _gpu_busy():
    """True if NVML lists a compute process on GPU 0 besides this one (the rule b2dp_int_test applies)."""
    try:
        import pynvml
        pynvml.nvmlInit()
        return len(pynvml.nvmlDeviceGetComputeRunningProcesses(pynvml.nvmlDeviceGetHandleByIndex(0))) > 1
    except Exception:       # noqa: BLE001
        return None


def launch_tables(seed, fmt):
    """The launch inputs from the oracle: tables (TILES x SLOTS x THREADS words) and checks (TILES x THREADS)."""
    tables = np.array([it.table(seed, fmt, t) for t in range(it.TILES)], dtype=np.uint32)
    checks = np.array([it.tile_checks(seed, fmt, t) for t in range(it.TILES)], dtype=np.uint32)
    return tables.reshape(it.TILES, it.SLOTS[fmt], it.THREADS), checks


# ---- the kernel, directly ---------------------------------------------------------------------------------------------
@pytest.mark.parametrize("seed", [0x0, 0xC0FFEE17])
@pytest.mark.parametrize("fmt", FORMATS, ids=FMT_IDS)
def test_dump_matches_the_oracle_word_for_word(H, fmt, seed):
    got, rec = H.dump(fmt, seed)
    bad = []
    for t in range(it.TILES):
        want = np.array(it.tile_words(seed, fmt, t), dtype=np.uint32)
        if not np.array_equal(got[t], want):
            idx = np.argwhere(got[t] != want)
            names = sorted({it.WORD_NAMES[fmt][j % it.SET_WORDS[fmt]] for _, j in idx})
            th, j = idx[0]
            bad.append("tile %d: %d of %d words differ (%s); first thread %d word %d got 0x%08x want 0x%08x"
                       % (t, len(idx), want.size, ",".join(names), th, j, got[t][th, j], want[th, j]))
    assert not bad, "\n".join(bad)
    assert (rec.seq, rec.rounds, rec.comparisons, rec.mismatches) == (7, 1, it.TILES * it.REPS, 0), \
        (rec.seq, rec.rounds, rec.comparisons, rec.mismatches)
    assert (rec.first_bad_tile, rec.first_bad_rep) == (-1, -1)


def _check_clean(recs, seq=7):
    for r in recs:
        assert r.seq == seq and r.rounds >= 1 and r.comparisons == r.rounds * it.TILES * it.REPS, \
            (r.smid, r.seq, r.rounds, r.comparisons)
        assert r.mismatches == 0 and (r.first_bad_tile, r.first_bad_rep) == (-1, -1), \
            (r.smid, r.mismatches, r.first_bad_tile, r.first_bad_rep)
        assert r.smid < r.nsmid <= 256


@pytest.fixture(scope="module")
def sm_ids(H):
    recs, _ = H.run(it.BIT, 0x5EED, 20)
    _check_clean(recs)
    return sorted({r.smid for r in recs})


@pytest.mark.parametrize("fmt", FORMATS, ids=FMT_IDS)
def test_clean_run_covers_every_sm(H, fmt):
    duration = 100
    recs, ms = H.run(fmt, 0x1234567 + fmt, duration)
    assert len(recs) == H.sms * H.occupancy(fmt)
    _check_clean(recs)
    assert ms >= duration * 0.9
    results = it.THREADS * it.WORDS[fmt] * sum(r.comparisons for r in recs)
    print("%s: %d CTAs (%d resident per SM), %d SM ids, %.1f ms, %.2f T results/s"
          % (FMT_IDS[fmt], len(recs), H.occupancy(fmt), len({r.smid for r in recs}), ms, results / ms * 1e-9))
    if _gpu_busy():
        pytest.skip("another process uses the GPU: coverage is not asserted (the rest was)")
    assert len({r.smid for r in recs}) == H.sms


@pytest.mark.parametrize("fmt", FORMATS, ids=FMT_IDS)
def test_32_seeds_run_clean_on_a_full_grid(H, fmt):
    for k in range(32):
        recs, _ = H.run(fmt, (0x9E3779B9 * (k + 1) + fmt) & 0xFFFFFFFF, 1)
        assert len(recs) == H.sms * H.occupancy(fmt)
        _check_clean(recs)


@pytest.mark.parametrize("fmt", FORMATS, ids=FMT_IDS)
def test_wrong_check_value_in_every_thread_is_counted_in_its_tile(H, fmt):
    tables, checks = launch_tables(0xC4EC, fmt)
    for t in range(it.THREADS):
        tile = t % it.TILES
        bad = checks.copy()
        bad[tile, t] ^= np.uint32(1 << (t % 32))
        (r,) = H.run_tables(fmt, tables, bad)
        assert (r.seq, r.rounds, r.comparisons) == (7, 1, it.TILES * it.REPS)
        assert (r.mismatches, r.first_bad_tile, r.first_bad_rep) == (it.REPS, tile, 0), (t, r.mismatches, r.first_bad_tile)


# (fmt, tile, thread, set, k, bit): one operand word that each op family reads, in several warps.  The sets are random
# ones, so the flipped bit reaches a result word.
OPERAND_CASES = [
    (it.MAD, 0, 0, 16, 0, 5), (it.MAD, 3, 77, 17, 1, 22), (it.MAD, 5, 100, 18, 2, 0), (it.MAD, 7, 127, 19, 3, 31),
    (it.BIT, 1, 33, 11, 0, 17), (it.BIT, 4, 64, 11, 1, 3), (it.BIT, 6, 96, 11, 2, 2),
    (it.WARP, 0, 5, 4, 0, 9), (it.WARP, 2, 40, 4, 1, 0), (it.WARP, 3, 70, 7, 2, 12), (it.WARP, 4, 99, 6, 3, 0),
    (it.WARP, 5, 127, 6, 4, 30), (it.WARP, 6, 1, 0, 5, 7), (it.WARP, 7, 64, 0, 6, 19),
]


@pytest.mark.parametrize("fmt,tile,thread,s,k,bit", OPERAND_CASES)
def test_wrong_operand_is_counted_in_every_repetition_of_every_round_by_every_cta(H, fmt, tile, thread, s, k, bit):
    tables, checks = launch_tables(0x0BAD, fmt)
    tables = tables.copy()
    tables[tile, s * it.SET_SLOTS[fmt] + k, thread] ^= np.uint32(1 << bit)
    grid = H.sms * H.occupancy(fmt)
    recs = H.run_tables(fmt, tables, checks, grid=grid, duration_ms=10)
    assert len(recs) == grid
    for r in recs:
        assert r.seq == 7 and r.comparisons == r.rounds * it.TILES * it.REPS
        assert (r.mismatches, r.first_bad_tile, r.first_bad_rep) == (r.rounds * it.REPS, tile, 0), \
            (r.smid, r.rounds, r.mismatches, r.first_bad_tile)


FAULT_SAMPLE = [  # one model per op family; each changes a check in every tile (tests/test_int_test_cpu.py)
    (it.MAD, ("mulhi_unsigned",)), (it.MAD, ("column", 40)), (it.MAD, ("carry", 32)), (it.MAD, ("dp4a_sat",)),
    (it.BIT, ("lop3_minterm", 3)), (it.BIT, ("shift_stage", 4)), (it.BIT, ("clz0",)), (it.BIT, ("cmp_swapped",)),
    (it.WARP, ("segment_ignored",)), (it.WARP, ("pred_true",)), (it.WARP, ("redux_skip", 13)),
    (it.WARP, ("match_miss", 7)),
]


@pytest.mark.parametrize("fmt,fault", FAULT_SAMPLE, ids=["-".join(map(str, f)) for _, f in FAULT_SAMPLE])
def test_checks_of_a_faulty_unit_mismatch_in_every_tile(H, fmt, fault):
    seed = 0x1EEE
    tables, checks = launch_tables(seed, fmt)
    wrong = np.array([it.tile_checks(seed, fmt, t, fault) for t in range(it.TILES)], dtype=np.uint32)
    assert all((wrong[t] != checks[t]).any() for t in range(it.TILES))
    for r in H.run_tables(fmt, tables, wrong, grid=4):
        assert (r.rounds, r.mismatches, r.first_bad_tile, r.first_bad_rep) == (1, it.TILES * it.REPS, 0, 0), \
            (r.rounds, r.mismatches)
    _check_clean(H.run_tables(fmt, tables, checks, grid=4))


def test_run_tables_refuses_malformed_input(H):
    tables, checks = launch_tables(0, it.BIT)
    assert H.run_tables_rc(3, tables, checks)[0] == -1
    assert H.run_tables_rc(it.BIT, tables, checks, table_bytes=tables.nbytes - 4)[0] == -3
    assert H.run_tables_rc(it.MAD, tables, checks)[0] == -3
    assert H.run_tables_rc(it.BIT, tables, checks, n_checks=checks.size - 1)[0] == -3
    assert H.run_tables_rc(it.BIT, tables, checks, grid=0)[0] == -4
    assert H.run_tables_rc(it.BIT, tables, checks, grid=H.sms * 64)[0] == -4


# ---- through the ABI --------------------------------------------------------------------------------------------------
def _open(pkg, nbytes=64 * MiB):
    return pkg.Context("cuda:devices=0,bytes=%d,calib=1" % nbytes)


def test_int_test_clean_and_memory_back(pkg):
    import torch
    torch.cuda.init()
    N = pkg._native
    with _open(pkg) as ctx:
        ctx.int_test(0, duration_ms=10)                         # first launch loads the kernels: not counted below
        free0, _ = torch.cuda.mem_get_info(0)
        (r,) = ctx.int_test(0, duration_ms=100)
        free1, _ = torch.cuda.mem_get_info(0)
        assert r.healthy and r.err == 0, r
        assert r.mismatches == [0, 0, 0] and r.bad_sm_mask == [0, 0, 0, 0], r
        assert (r.first_bad_sm, r.first_bad_format, r.first_bad_tile) == (-1, -1, -1)
        assert r.sm_count == torch.cuda.get_device_properties(0).multi_processor_count
        assert r.nsmid >= r.sm_count and all(ms >= 90 for ms in r.ms) and all(t > 0 for t in r.tflops), r
        if not _gpu_busy():
            assert r.sms_covered == r.sm_count and r.flags == 0, r
        assert abs(free1 - free0) < 2 * MiB, (free0, free1)
        (p,) = ctx.probe_health(min_gbs=1e-3)
        assert p.healthy and not p.flags & N.RES_COMPUTE
    print("int test 100 ms/format: SMs %d/%d, ms %s, T results/s mad %.2f bit %.2f warp %.2f"
          % (r.sms_covered, r.sm_count, ["%.1f" % x for x in r.ms], *r.tflops))


@pytest.mark.parametrize("where,mask", [("first", 0x1), ("middle", 0x80000000), ("last", 0xFFFFFFFF)])
def test_int_test_fault_is_attributed_and_latched_until_reset(pkg, H, sm_ids, where, mask):
    N = pkg._native
    s = {"first": sm_ids[0], "middle": sm_ids[len(sm_ids) // 2], "last": sm_ids[-1]}[where]
    with _open(pkg) as ctx:
        (r,) = ctx.int_test(0, duration_ms=10, fault_sm=s, fault_mask=mask)
        assert not r.healthy and r.err == 0, r
        assert r.bad_sms() == [s], r.bad_sms()
        assert (r.first_bad_sm, r.first_bad_format, r.first_bad_tile) == (s, N.IT_MAD, 0), r
        for f in FORMATS:          # one mismatch per CTA that ran on s
            assert 1 <= r.mismatches[f] <= H.occupancy(f), (f, r.mismatches)
        (p,) = ctx.probe_health(min_gbs=1e-3)
        assert p.flags & N.RES_COMPUTE and p.flags & 0x400 and not p.healthy and p.mismatches == 0
        _, st = ctx.list_and_watch("gpu", N.LW_HEARTBEAT, min_gbs=1e-3)
        assert st.n_unhealthy == 1
        ctx.probe_reset(0)
        (p,) = ctx.probe_health(min_gbs=1e-3)
        assert p.healthy and not p.flags & N.RES_COMPUTE


def test_int_test_skips_a_busy_gpu(pkg):
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
            (r,) = ctx.int_test(0, duration_ms=10, fault_sm=0, fault_mask=1)
            assert r.flags & N.CT_SKIPPED_BUSY and r.mismatches == [0, 0, 0] and r.ms == [0, 0, 0], r
            (p,) = ctx.probe_health(min_gbs=1e-3)
            assert not p.flags & N.RES_COMPUTE
            (r,) = ctx.int_test(0, duration_ms=10, even_if_busy=True)
            assert not r.flags & N.CT_SKIPPED_BUSY and r.healthy and r.err == 0, r
    finally:
        if helper.poll() is None:
            helper.kill()
        helper.wait()


def _daemon_lines(short_dir, level):
    exe = os.path.join(ROOT, "k8s-device-plugin_b200", "b200dp_plugind")
    proc = subprocess.Popen([exe, "-backend=cuda:devices=0,bytes=67108864,calib=1", "-plugin_dir", short_dir,
                             "-start_retry_wait=0.05", "-int_test_at_start=%d" % level, "-compute_test_ms=50"],
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
    assert log.index("int test ") < log.index("Failed to start plugin"), log[-3000:]  # before the first registration
    return [ln for ln in log.splitlines() if ln.startswith("int test ")], log


def test_daemon_int_test_at_start_logs_a_clean_result(short_dir):
    lines, log = _daemon_lines(short_dir, 1)
    assert len(lines) == 1, log[-3000:]
    if "flags 0x1," in lines[0]:
        lines, log = _daemon_lines(short_dir, 2)
        assert len(lines) == 1, log[-3000:]
    assert ": Healthy, flags 0x" in lines[0] and "mismatches 0/0/0, first bad SM -1" in lines[0], log[-3000:]
