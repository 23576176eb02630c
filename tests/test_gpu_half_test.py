"""The on-demand half-precision and conversion self-test on a real H100.

- The kernel of half_selftest.cuh, launched directly (tests/native/libhalf_test_kernels_test.so):
  - the DUMP instantiation's result words equal tests/half_test_oracle.py word for word, for every format and tile at two
    seeds: this H100's 16-bit pipes and converters agree with the PTX ISA on every crafted class;
  - a clean run covers every SM id and every CTA compares exactly what its rounds hold, at 32 seeds per format through
    the product's table builder;
  - on caller-built tables: a wrong check value in any of the 128 threads is counted in exactly its tile's 16
    repetitions; a changed operand word in every repetition of every round by every CTA; and check values computed by
    a fault model of tests/test_half_test_cpu.py mismatch in the tiles the model says;
  - malformed tables are refused before anything runs.
- b2dp_half_test through the ABI: Healthy on an idle card, the fault hook attributed to its SM and latched until
  probe_reset, the busy skip, and the daemon's -half_test_at_start.

Every run is short: 0-100 ms per format."""
import ctypes as C
import os
import signal
import subprocess
import sys
import time

import numpy as np
import pytest

import half_test_oracle as it

pytestmark = pytest.mark.gpu

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(HERE)
LIB_PATH = os.path.join(HERE, "native", "libhalf_test_kernels_test.so")
MiB = 1 << 20
MS = 1000000
FORMATS = (it.F16, it.BF16, it.CVT)
FMT_IDS = ["f16", "bf16", "cvt"]


class CtRecord(C.Structure):
    _fields_ = [("smid", C.c_uint32), ("nsmid", C.c_uint32), ("rounds", C.c_uint64), ("comparisons", C.c_uint64),
                ("mismatches", C.c_uint64), ("first_bad_tile", C.c_int32), ("first_bad_rep", C.c_int32),
                ("seq", C.c_uint64)]


_P = C.POINTER


class Harness:
    def __init__(self, device=0):
        L = C.CDLL(LIB_PATH)
        L.hk_open.restype = C.c_void_p
        L.hk_open.argtypes = [C.c_int, C.c_char_p, C.c_int]
        L.hk_close.argtypes = [C.c_void_p]
        L.hk_error.restype = C.c_char_p
        L.hk_error.argtypes = [C.c_void_p]
        L.hk_sms.argtypes = [C.c_void_p]
        L.hk_table_bytes.restype = C.c_uint64
        L.hk_occupancy.argtypes = [C.c_void_p, C.c_int, _P(C.c_int)]
        L.hk_dump.argtypes = [C.c_void_p, C.c_int, C.c_uint32, _P(C.c_uint32), _P(CtRecord)]
        L.hk_run.argtypes = [C.c_void_p, C.c_int, C.c_uint32, C.c_uint64, C.c_int, C.c_uint32, _P(CtRecord), C.c_int,
                             _P(C.c_int), _P(C.c_float)]
        L.hk_run_tables.argtypes = [C.c_void_p, C.c_int, C.c_int, C.c_void_p, C.c_uint64, C.c_void_p, C.c_uint64,
                                    C.c_int, C.c_uint64, _P(CtRecord), C.c_int, _P(C.c_int), _P(C.c_float),
                                    _P(C.c_uint32)]
        assert L.hk_record_bytes() == C.sizeof(CtRecord)
        assert (L.hk_tiles(), L.hk_reps()) == (it.TILES, it.REPS)
        assert [L.hk_words(f) for f in FORMATS] == list(it.WORDS)
        assert [L.hk_table_bytes(f) for f in FORMATS] == [4 * it.THREADS * s for s in it.SLOTS]
        self.L = L
        err = C.create_string_buffer(512)
        self.h = L.hk_open(device, err, len(err))
        if not self.h:
            raise RuntimeError("hk_open: " + err.value.decode())
        self.sms = L.hk_sms(self.h)

    def close(self):
        if self.h:
            self.L.hk_close(self.h)
            self.h = None

    def _check(self, rc, what):
        if rc == 1:
            raise RuntimeError("%s: %s" % (what, self.L.hk_error(self.h).decode()))
        assert rc == 0, "%s refused: code %d" % (what, rc)

    def occupancy(self, fmt):
        n = C.c_int()
        self._check(self.L.hk_occupancy(self.h, fmt, C.byref(n)), "hk_occupancy")
        return n.value

    def dump(self, fmt, seed):
        out = np.zeros(it.TILES * it.THREADS * it.WORDS[fmt], dtype=np.uint32)
        rec = CtRecord()
        self._check(self.L.hk_dump(self.h, fmt, seed, out.ctypes.data_as(_P(C.c_uint32)), C.byref(rec)), "hk_dump")
        return out.reshape(it.TILES, it.THREADS, it.WORDS[fmt]), rec

    def run(self, fmt, seed, duration_ms, fault_sm=-1, fault_mask=0):
        cap = self.sms * 32
        recs = (CtRecord * cap)()
        n, ms = C.c_int(), C.c_float()
        self._check(self.L.hk_run(self.h, fmt, seed, int(duration_ms * MS), fault_sm, fault_mask, recs, cap,
                                  C.byref(n), C.byref(ms)), "hk_run")
        return list(recs[:n.value]), ms.value

    def run_tables_rc(self, fmt, tables, checks, grid=1, duration_ms=0, table_bytes=None, n_checks=None):
        cap = max(grid, 1)
        recs = (CtRecord * cap)()
        n, ms = C.c_int(), C.c_float()
        rc = self.L.hk_run_tables(self.h, fmt, 0, tables.ctypes.data, tables.nbytes if table_bytes is None
                                  else table_bytes, checks.ctypes.data, checks.size if n_checks is None else n_checks,
                                  grid, int(duration_ms * MS), recs, cap, C.byref(n), C.byref(ms), None)
        return rc, list(recs[:n.value]) if rc == 0 else []

    def run_tables(self, fmt, tables, checks, grid=1, duration_ms=0):
        rc, recs = self.run_tables_rc(fmt, tables, checks, grid, duration_ms)
        self._check(rc, "hk_run_tables")
        return recs


@pytest.fixture(scope="module")
def H():
    if not os.path.exists(LIB_PATH):
        pytest.skip("run __graft_entry__.build() first")
    h = Harness(0)
    yield h
    h.close()


def _gpu_busy():
    """True if NVML lists a compute process on GPU 0 besides this one (the rule b2dp_half_test applies)."""
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
            rows = []
            for th, j in idx[:12]:
                s, k = divmod(j, it.SET_WORDS[fmt])
                rows.append("  thread %d set %d %s got 0x%08x want 0x%08x operands %s"
                            % (th, s, it.WORD_NAMES[fmt][k], got[t][th, j], want[th, j],
                               ",".join("%08x" % x for x in it.tile_operands(seed, fmt, t)[th][s])))
            bad.append("tile %d: %d of %d words differ (%s)\n%s" % (t, len(idx), want.size, ",".join(names),
                                                                   "\n".join(rows)))
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
    recs, _ = H.run(it.BF16, 0x5EED, 20)
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


# (fmt, tile, thread, set, k, bit): one operand word of a random set, in several warps.  Each flip provably changes a
# result word whatever the random values: a lane's sign into min / max or min.xorsign.abs, an f32's sign into a pack
# (-0 and +0 differ) or into rmi / rpi, 2^25 into an s32 converted to f32, a kept f64 significand bit into f32.
OPERAND_CASES = [
    (it.F16, 0, 0, 7, 3, 15), (it.F16, 3, 77, 9, 4, 31), (it.F16, 6, 127, 11, 0, 15),
    (it.BF16, 1, 33, 6, 3, 15), (it.BF16, 5, 100, 10, 4, 31),
    (it.CVT, 0, 5, 8, 0, 31), (it.CVT, 2, 40, 8, 4, 31), (it.CVT, 4, 64, 8, 5, 15), (it.CVT, 5, 99, 8, 8, 25),
    (it.CVT, 7, 127, 8, 10, 1),
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


FAULT_SAMPLE = [  # one model per unit behaviour; each changes checks in every tile (tests/test_half_test_cpu.py)
    (it.F16, "lane_swap"), (it.F16, "sticky_lost"), (it.F16, "sat_ignored"), (it.F16, "double_round"),
    (it.BF16, "rz"), (it.BF16, "relu_ignored"),
    (it.CVT, "fp8_order"), (it.CVT, "satfinite_ignored"), (it.CVT, "nan_not_zero"), (it.CVT, "i2f_rn"),
    (it.CVT, "frnd_trunc"),
]


@pytest.mark.parametrize("fmt,fault", FAULT_SAMPLE, ids=["%s-%s" % (FMT_IDS[f], m) for f, m in FAULT_SAMPLE])
def test_checks_of_a_faulty_unit_mismatch_in_the_tiles_the_model_names(H, fmt, fault):
    seed = 0x1EEE
    tables, checks = launch_tables(seed, fmt)
    wrong = np.array([it.tile_checks(seed, fmt, t, fault) for t in range(it.TILES)], dtype=np.uint32)
    tiles = [t for t in range(it.TILES) if (wrong[t] != checks[t]).any()]
    assert tiles == list(range(it.TILES))
    for r in H.run_tables(fmt, tables, wrong, grid=4):
        assert (r.rounds, r.mismatches, r.first_bad_tile, r.first_bad_rep) == (1, it.TILES * it.REPS, 0, 0), \
            (r.rounds, r.mismatches)
    _check_clean(H.run_tables(fmt, tables, checks, grid=4))


def test_run_tables_refuses_malformed_input(H):
    tables, checks = launch_tables(0, it.BF16)
    assert H.run_tables_rc(3, tables, checks)[0] == -1
    assert H.run_tables_rc(it.BF16, tables, checks, table_bytes=tables.nbytes - 4)[0] == -3
    assert H.run_tables_rc(it.CVT, tables, checks)[0] == -3
    assert H.run_tables_rc(it.BF16, tables, checks, n_checks=checks.size - 1)[0] == -3
    assert H.run_tables_rc(it.BF16, tables, checks, grid=0)[0] == -4
    assert H.run_tables_rc(it.BF16, tables, checks, grid=H.sms * 64)[0] == -4


# ---- through the ABI --------------------------------------------------------------------------------------------------
def _open(pkg, nbytes=64 * MiB):
    return pkg.Context("cuda:devices=0,bytes=%d,calib=1" % nbytes)


def test_half_test_clean_and_memory_back(pkg):
    import torch
    torch.cuda.init()
    N = pkg._native
    with _open(pkg) as ctx:
        ctx.half_test(0, duration_ms=10)                         # first launch loads the kernels: not counted below
        free0, _ = torch.cuda.mem_get_info(0)
        (r,) = ctx.half_test(0, duration_ms=100)
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
    print("half test 100 ms/format: SMs %d/%d, ms %s, T results/s f16 %.2f bf16 %.2f cvt %.2f"
          % (r.sms_covered, r.sm_count, ["%.1f" % x for x in r.ms], *r.tflops))


@pytest.mark.parametrize("where,mask", [("first", 0x1), ("middle", 0x80000000), ("last", 0xFFFFFFFF)])
def test_half_test_fault_is_attributed_and_latched_until_reset(pkg, H, sm_ids, where, mask):
    N = pkg._native
    s = {"first": sm_ids[0], "middle": sm_ids[len(sm_ids) // 2], "last": sm_ids[-1]}[where]
    with _open(pkg) as ctx:
        (r,) = ctx.half_test(0, duration_ms=10, fault_sm=s, fault_mask=mask)
        assert not r.healthy and r.err == 0, r
        assert r.bad_sms() == [s], r.bad_sms()
        assert (r.first_bad_sm, r.first_bad_format, r.first_bad_tile) == (s, N.HP_F16, 0), r
        for f in FORMATS:          # one mismatch per CTA that ran on s
            assert 1 <= r.mismatches[f] <= H.occupancy(f), (f, r.mismatches)
        (p,) = ctx.probe_health(min_gbs=1e-3)
        assert p.flags & N.RES_COMPUTE and p.flags & 0x400 and not p.healthy and p.mismatches == 0
        _, st = ctx.list_and_watch("gpu", N.LW_HEARTBEAT, min_gbs=1e-3)
        assert st.n_unhealthy == 1
        ctx.probe_reset(0)
        (p,) = ctx.probe_health(min_gbs=1e-3)
        assert p.healthy and not p.flags & N.RES_COMPUTE


def test_half_test_skips_a_busy_gpu(pkg):
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
            (r,) = ctx.half_test(0, duration_ms=10, fault_sm=0, fault_mask=1)
            assert r.flags & N.CT_SKIPPED_BUSY and r.mismatches == [0, 0, 0] and r.ms == [0, 0, 0], r
            (p,) = ctx.probe_health(min_gbs=1e-3)
            assert not p.flags & N.RES_COMPUTE
            (r,) = ctx.half_test(0, duration_ms=10, even_if_busy=True)
            assert not r.flags & N.CT_SKIPPED_BUSY and r.healthy and r.err == 0, r
    finally:
        if helper.poll() is None:
            helper.kill()
        helper.wait()


def _daemon_lines(short_dir, level):
    exe = os.path.join(ROOT, "k8s-device-plugin_b200", "b200dp_plugind")
    proc = subprocess.Popen([exe, "-backend=cuda:devices=0,bytes=67108864,calib=1", "-plugin_dir", short_dir,
                             "-start_retry_wait=0.05", "-half_test_at_start=%d" % level, "-compute_test_ms=50"],
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
    assert log.index("half test ") < log.index("Failed to start plugin"), log[-3000:]  # before the first registration
    return [ln for ln in log.splitlines() if ln.startswith("half test ")], log


def test_daemon_half_test_at_start_logs_a_clean_result(short_dir):
    lines, log = _daemon_lines(short_dir, 1)
    assert len(lines) == 1, log[-3000:]
    if "flags 0x1," in lines[0]:
        lines, log = _daemon_lines(short_dir, 2)
        assert len(lines) == 1, log[-3000:]
    assert ": Healthy, flags 0x" in lines[0] and "mismatches 0/0/0, first bad SM -1" in lines[0], log[-3000:]
