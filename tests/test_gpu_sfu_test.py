"""The on-demand SFU self-test on a real H100.

- The premise: every SM's special-function unit returns the same bits for the same operands.  At 64 seeds per format
  the reference launch (one CTA on every SM) is unanimous, and its words pass the guard of tests/sfu_test_oracle.py;
  the worst observed error per op is printed.  Two fixed seeds' words match tests/golden/sfu_sm90_consensus.json
  (captured on an H100 by tools/sfu_consensus_golden.py), which pins later cards, drivers and kernel edits to them.
- The kernel of sfu_selftest.cuh, launched directly (tests/native/libsfu_test_kernels_test.so): the reference launch
  puts exactly one CTA on each SM id; on caller-built tables a wrong check value in each of the 128 threads is counted in
  exactly its tile's 16 repetitions, and a changed operand of each op in every repetition of every round by every CTA;
  malformed tables are refused.
- b2dp_sfu_test through the ABI: Healthy on an idle card with every SM id covered, memory handed back, the probe ring
  untouched; the fault hook on the first, middle and last SM id attributed to that SM alone, latched until probe_reset;
  the busy skip; the daemon's -sfu_test_at_start."""
import ctypes as C
import hashlib
import json
import os
import signal
import subprocess
import sys
import time

import numpy as np
import pytest

import sfu_test_oracle as so
from oracle import probe as oprobe

pytestmark = pytest.mark.gpu

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(HERE)
LIB_PATH = os.path.join(HERE, "native", "libsfu_test_kernels_test.so")
GOLDEN = os.path.join(HERE, "golden", "sfu_sm90_consensus.json")
MiB = 1 << 20
MS = 1000000
FMT_IDS = [so.NAMES[f] for f in so.FORMATS]
_P = C.POINTER


class CtRecord(C.Structure):
    _fields_ = [("smid", C.c_uint32), ("nsmid", C.c_uint32), ("rounds", C.c_uint64), ("comparisons", C.c_uint64),
                ("mismatches", C.c_uint64), ("first_bad_tile", C.c_int32), ("first_bad_rep", C.c_int32),
                ("seq", C.c_uint64)]


class Harness:
    def __init__(self, device=0):
        L = C.CDLL(LIB_PATH)
        L.sk_open.restype = C.c_void_p
        L.sk_open.argtypes = [C.c_int, C.c_char_p, C.c_int]
        L.sk_close.argtypes = [C.c_void_p]
        L.sk_error.restype = C.c_char_p
        L.sk_error.argtypes = [C.c_void_p]
        L.sk_sms.argtypes = [C.c_void_p]
        L.sk_occupancy.argtypes = [C.c_void_p, C.c_int, C.c_int, _P(C.c_int)]
        L.sk_tables.argtypes = [C.c_int, C.c_uint32, _P(C.c_uint32)]
        L.sk_dump.argtypes = [C.c_void_p, C.c_int, C.c_uint32, C.c_int, C.c_uint32, _P(C.c_uint32), _P(CtRecord),
                              C.c_int, _P(C.c_int), _P(C.c_float)]
        L.sk_run.argtypes = [C.c_void_p, C.c_int, C.c_uint32, C.c_uint64, C.c_int, C.c_uint32, _P(CtRecord), C.c_int,
                             _P(C.c_int), _P(C.c_float), _P(C.c_double)]
        L.sk_run_tables.argtypes = [C.c_void_p, C.c_int, C.c_int, C.c_void_p, C.c_uint64, C.c_void_p, C.c_uint64,
                                    C.c_int, C.c_uint64, _P(CtRecord), C.c_int, _P(C.c_int), _P(C.c_float),
                                    _P(C.c_uint32)]
        assert L.sk_record_bytes() == C.sizeof(CtRecord)
        assert (L.sk_tiles(), L.sk_reps()) == (so.TILES, so.REPS)
        assert [L.sk_words(f) for f in so.FORMATS] == [so.WORDS[f] for f in so.FORMATS]
        assert [L.sk_slots(f) for f in so.FORMATS] == [so.SLOTS[f] for f in so.FORMATS]
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

    def occupancy(self, fmt, dump=False):
        n = C.c_int()
        self._check(self.L.sk_occupancy(self.h, fmt, int(dump), C.byref(n)), "sk_occupancy")
        return n.value

    def tables(self, fmt, seed):
        out = np.zeros((so.TILES, so.SLOTS[fmt], so.THREADS), dtype=np.uint32)
        assert self.L.sk_tables(fmt, seed, out.ctypes.data_as(_P(C.c_uint32))) == 0
        return out

    def dump(self, fmt, seed, fault_sm=-1, fault_mask=0):
        """The reference launch: ([cta][tile][thread][word] words, records, ms)."""
        out = np.zeros((self.sms, so.TILES, so.THREADS, so.WORDS[fmt]), dtype=np.uint32)
        recs = (CtRecord * self.sms)()
        n, ms = C.c_int(), C.c_float()
        self._check(self.L.sk_dump(self.h, fmt, seed, fault_sm, fault_mask, out.ctypes.data_as(_P(C.c_uint32)), recs,
                                   self.sms, C.byref(n), C.byref(ms)), "sk_dump")
        return out, list(recs[:n.value]), ms.value

    def run(self, fmt, seed, duration_ms, fault_sm=-1, fault_mask=0):
        cap = self.sms * 32
        recs = (CtRecord * cap)()
        n, ms = C.c_int(), C.c_float()
        info = (C.c_double * 3)()
        self._check(self.L.sk_run(self.h, fmt, seed, int(duration_ms * MS), fault_sm, fault_mask, recs, cap,
                                  C.byref(n), C.byref(ms), info), "sk_run")
        return list(recs[:n.value]), ms.value, list(info)

    def run_tables_rc(self, fmt, tables, checks, grid=1, duration_ms=0, dump=False, table_bytes=None, n_checks=None):
        cap = max(grid, 1)
        recs = (CtRecord * cap)()
        n, ms = C.c_int(), C.c_float()
        out = np.zeros((cap, so.TILES, so.THREADS, so.WORDS[fmt]), dtype=np.uint32) if dump else None
        rc = self.L.sk_run_tables(self.h, fmt, int(dump), tables.ctypes.data, tables.nbytes if table_bytes is None
                                  else table_bytes, checks.ctypes.data, checks.size if n_checks is None else n_checks,
                                  grid, int(duration_ms * MS), recs, cap, C.byref(n), C.byref(ms),
                                  out.ctypes.data_as(_P(C.c_uint32)) if dump else None)
        return rc, list(recs[:n.value]) if rc == 0 else [], out

    def run_tables(self, fmt, tables, checks, grid=1, duration_ms=0, dump=False):
        rc, recs, out = self.run_tables_rc(fmt, tables, checks, grid, duration_ms, dump)
        self._check(rc, "sk_run_tables")
        return (recs, out) if dump else recs


@pytest.fixture(scope="module")
def H():
    if not os.path.exists(LIB_PATH):
        pytest.skip("run __graft_entry__.build() first")
    h = Harness(0)
    yield h
    h.close()


def _gpu_busy():
    """True if NVML lists a compute process on GPU 0 besides this one (the rule b2dp_sfu_test applies)."""
    try:
        import pynvml
        pynvml.nvmlInit()
        return len(pynvml.nvmlDeviceGetComputeRunningProcesses(pynvml.nvmlDeviceGetHandleByIndex(0))) > 1
    except Exception:       # noqa: BLE001
        return None


def _arrived(recs, seq=7):
    for r in recs:
        assert r.seq == seq and r.rounds >= 1 and r.comparisons == r.rounds * so.TILES * so.REPS, \
            (r.smid, r.seq, r.rounds, r.comparisons)
        assert r.smid < r.nsmid <= 256


def _check_clean(recs, seq=7):
    _arrived(recs, seq)
    for r in recs:
        assert r.mismatches == 0 and (r.first_bad_tile, r.first_bad_rep) == (-1, -1), (r.smid, r.mismatches)


_CONS = {}


def consensus(H, fmt, seed):
    """(tables, majority words [tile][thread][word], checks [tile][thread]) of one seed on this GPU, cached.  The
    reference launch must be unanimous (the premise)."""
    if (fmt, seed) not in _CONS:
        d, recs, _ = H.dump(fmt, seed)
        _arrived(recs)
        assert (d == d[0][None]).all(), "the SMs disagree"
        _CONS[fmt, seed] = (H.tables(fmt, seed), d[0].copy(), so.fold(d[0]))
    return _CONS[fmt, seed]


# ---- the premise --------------------------------------------------------------------------------------------------------
def test_reference_launch_puts_one_cta_on_each_sm(H):
    for fmt in so.FORMATS:
        assert H.occupancy(fmt, dump=True) == 1
        _, recs, ms = H.dump(fmt, 0x51D)
        _arrived(recs)
        assert len(recs) == H.sms
        print("%s reference launch: %d CTAs on %d SM ids, %.2f ms" % (so.NAMES[fmt], len(recs),
                                                                     len({r.smid for r in recs}), ms))
        if _gpu_busy():
            pytest.skip("another process uses the GPU: coverage is not asserted")
        assert sorted(r.smid for r in recs) == sorted(set(r.smid for r in recs)) and len(recs) == H.sms


@pytest.mark.parametrize("fmt", so.FORMATS, ids=FMT_IDS)
def test_every_sm_agrees_bit_for_bit_and_the_majority_passes_the_guard(H, fmt):
    """64 seeds: every result word of every tile and thread, on every SM, equals SM 0's; the words pass the guard."""
    worst, disagree = {}, []
    for seed in range(1000, 1064):
        d, recs, _ = H.dump(fmt, seed)
        _arrived(recs)
        same = (d == d[0][None]).reshape(len(recs), -1).all(axis=1)
        if not same.all():
            med, has = so.majority(d)
            for c in np.nonzero(~same)[0]:
                idx = np.argwhere(d[c] != med)[0]
                disagree.append("seed %d SM %d: %d words differ from the majority, first [tile, thread, word] %s "
                                "got 0x%08x majority 0x%08x" % (seed, recs[c].smid, int((d[c] != med).sum()),
                                                               idx.tolist(), d[c][tuple(idx)], med[tuple(idx)]))
            if not has.all():
                disagree.append("seed %d: %d words without a majority" % (seed, int((~has).sum())))
            ref = med
        else:
            ref = d[0]
        tabs = H.tables(fmt, seed)
        ops = tabs.transpose(0, 2, 1)                    # [tile][thread][slot]
        bad, w = so.guard_words(fmt, ops, ref)
        assert bad == 0, (seed, bad)
        for k, v in w.items():
            worst[k] = max(worst.get(k, 0.0), v)
    for (op, fn), v in sorted(worst.items()):
        print("%s %s/%s worst guarded error %.3g (2^%.2f)" % (so.NAMES[fmt], op, fn, v, np.log2(v) if v else -np.inf))
    assert not disagree, "\n".join(disagree[:20])


def test_consensus_matches_the_golden_values(H):
    if not os.path.exists(GOLDEN):
        pytest.skip("no golden file")
    with open(GOLDEN) as f:
        gold = json.load(f)
    got = {}
    for seed in gold["seeds"]:
        for fmt in so.FORMATS:
            _, words, _ = consensus(H, fmt, seed)
            for t in range(so.TILES):
                got["%d/%s/%d" % (seed, so.NAMES[fmt], t)] = hashlib.sha256(words[t].tobytes()).hexdigest()
    bad = [k for k in gold["sha256"] if got.get(k) != gold["sha256"][k]]
    assert set(got) == set(gold["sha256"]) and not bad, bad


# ---- the kernel on caller-built tables ------------------------------------------------------------------------------
@pytest.mark.parametrize("fmt", so.FORMATS, ids=FMT_IDS)
def test_clean_timed_run_covers_every_sm(H, fmt):
    recs, ms, (flags, dissents, ref_ms) = H.run(fmt, 0x1234 + fmt, 100)
    assert (flags, dissents) == (0, 0)
    assert len(recs) == H.sms * H.occupancy(fmt)
    _check_clean(recs)
    assert ms >= 90
    results = so.THREADS * so.RESULTS[fmt] * sum(r.comparisons for r in recs)
    print("%s: %d CTAs (%d per SM), %.1f ms, %.2f T results/s; reference launch and consensus %.1f ms"
          % (so.NAMES[fmt], len(recs), H.occupancy(fmt), ms, results / ms * 1e-9, ref_ms))
    if not _gpu_busy():
        assert len({r.smid for r in recs}) == H.sms


@pytest.mark.parametrize("fmt", so.FORMATS, ids=FMT_IDS)
def test_wrong_check_value_in_every_thread_is_counted_in_its_tile(H, fmt):
    tables, _, checks = consensus(H, fmt, 0xC4EC)
    _check_clean(H.run_tables(fmt, tables, checks))
    for t in range(so.THREADS):
        tile = t % so.TILES
        bad = checks.copy()
        bad[tile, t] ^= np.uint32(1 << (t % 32))
        (r,) = H.run_tables(fmt, tables, bad)
        assert (r.seq, r.rounds, r.comparisons) == (7, 1, so.TILES * so.REPS)
        assert (r.mismatches, r.first_bad_tile, r.first_bad_rep) == (so.REPS, tile, 0), (t, r.mismatches)


def _changed_operand(H, fmt, op, tables, words, tile):
    """Tables with the top mantissa bit of one random-class operand of `op` flipped, chosen so that one CTA's result
    words change (checked with a DUMP launch): (tables, thread)."""
    name, _, T, _, s0, _, _, head, _ = so.OPS[op]
    nc, nv = len(head) + len(so.TAIL), so.values(op)
    M = so.BIN[T][1]
    for t in range(3, so.THREADS, 17):
        for v in range(nv):
            if (v - t) % nv < nc:
                continue
            bad = tables.copy()
            if T == so.T32:
                bad[tile, s0 + v, t] ^= np.uint32(1 << (M - 1))
            elif T == so.T64:
                bad[tile, s0 + 2 * v + 1, t] ^= np.uint32(1 << (M - 1 - 32))
            else:
                bad[tile, s0 + v // 2, t] ^= np.uint32(1 << (M - 1 + 16 * (v % 2)))
            _, out = H.run_tables(fmt, bad, so.fold(words), dump=True)
            if not np.array_equal(out[0, tile, t], words[tile, t]):
                return bad, t
    raise AssertionError("no operand of %s changes a result" % name)


@pytest.mark.parametrize("op", range(len(so.OPS)), ids=[o[0] for o in so.OPS])
def test_changed_operand_is_counted_in_every_repetition_of_every_round_by_every_cta(H, op):
    fmt = so.OPS[op][1]
    tables, words, checks = consensus(H, fmt, 0x0BAD)
    tile = op % so.TILES
    bad, _ = _changed_operand(H, fmt, op, tables, words, tile)
    grid = H.sms * H.occupancy(fmt)
    recs = H.run_tables(fmt, bad, checks, grid=grid, duration_ms=10)
    assert len(recs) == grid
    for r in recs:
        assert r.seq == 7 and r.comparisons == r.rounds * so.TILES * so.REPS
        assert (r.mismatches, r.first_bad_tile, r.first_bad_rep) == (r.rounds * so.REPS, tile, 0), \
            (r.smid, r.rounds, r.mismatches, r.first_bad_tile)


def test_run_tables_refuses_malformed_input(H):
    tables, _, checks = consensus(H, so.F32, 0xC4EC)
    assert H.run_tables_rc(3, tables, checks)[0] == -1
    assert H.run_tables_rc(so.F32, tables, checks, table_bytes=tables.nbytes - 4)[0] == -3
    assert H.run_tables_rc(so.ROOT, tables, checks)[0] == -3
    assert H.run_tables_rc(so.F32, tables, checks, n_checks=checks.size - 1)[0] == -3
    assert H.run_tables_rc(so.F32, tables, checks, grid=0)[0] == -4
    assert H.run_tables_rc(so.F32, tables, checks, grid=H.sms * 64)[0] == -4
    assert H.run_tables_rc(so.F32, tables, checks, grid=H.sms + 1, dump=True)[0] == -4


# ---- through the ABI --------------------------------------------------------------------------------------------------
def _open(pkg, nbytes=64 * MiB):
    return pkg.Context("cuda:devices=0,bytes=%d,calib=1" % nbytes)


@pytest.fixture(scope="module")
def sm_ids(H):
    _, recs, _ = H.dump(so.F32, 0x5EED)
    _arrived(recs)
    return sorted({r.smid for r in recs})


def test_sfu_test_clean_memory_back_and_ring_untouched(pkg):
    import torch
    torch.cuda.init()
    N = pkg._native
    nbytes = 64 * MiB
    n_words = nbytes // 4
    with _open(pkg, nbytes) as ctx:
        ctx.sfu_test(0, duration_ms=10)                        # first launch loads the kernels: not counted below
        (p0,) = ctx.probe_health(min_gbs=1e-3)
        seed = oprobe.next_seed(p0.seed)
        src = ctx.probe_peek(0, 0, n_words)
        free0, _ = torch.cuda.mem_get_info(0)
        (r,) = ctx.sfu_test(0, duration_ms=100)
        free1, _ = torch.cuda.mem_get_info(0)
        assert r.healthy and r.err == 0, r
        assert r.mismatches == [0, 0, 0] and r.bad_sm_mask == [0, 0, 0, 0], r
        assert not r.flags & (N.CT_NO_CONSENSUS | N.CT_OUT_OF_BOUND), r
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
    print("sfu test 100 ms/format: SMs %d/%d, ms %s, T results/s f32 %.2f root %.2f f16 %.2f"
          % (r.sms_covered, r.sm_count, ["%.1f" % x for x in r.ms], *r.tflops))


@pytest.mark.parametrize("where", ["first", "middle", "last"])
@pytest.mark.parametrize("mask", [0x1, 0x80000000])
def test_sfu_test_fault_is_attributed_and_latched_until_reset(pkg, H, sm_ids, where, mask):
    N = pkg._native
    s = {"first": sm_ids[0], "middle": sm_ids[len(sm_ids) // 2], "last": sm_ids[-1]}[where]
    with _open(pkg) as ctx:
        (r,) = ctx.sfu_test(0, duration_ms=10, fault_sm=s, fault_mask=mask)
        assert not r.healthy and r.err == 0, r
        assert r.bad_sms() == [s], r.bad_sms()
        assert (r.first_bad_sm, r.first_bad_format, r.first_bad_tile) == (s, N.SF_F32, 0), r
        assert not r.flags & (N.CT_NO_CONSENSUS | N.CT_OUT_OF_BOUND), r
        for f in so.FORMATS:      # the reference CTA on s dissents once, and every timed CTA on s mismatches once
            assert 2 <= r.mismatches[f] <= 1 + H.occupancy(f), (f, r.mismatches)
        (p,) = ctx.probe_health(min_gbs=1e-3)
        assert p.flags & N.RES_COMPUTE and not p.healthy and p.mismatches == 0
        _, st = ctx.list_and_watch("gpu", N.LW_HEARTBEAT, min_gbs=1e-3)
        assert st.n_unhealthy == 1
        ctx.probe_reset(0)
        (p,) = ctx.probe_health(min_gbs=1e-3)
        assert p.healthy and not p.flags & N.RES_COMPUTE
        (r,) = ctx.sfu_test(0, duration_ms=10)
        assert r.healthy and r.bad_sm_mask == [0, 0, 0, 0], r


def test_sfu_test_skips_a_busy_gpu(pkg):
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
            (r,) = ctx.sfu_test(0, duration_ms=10, fault_sm=0, fault_mask=1)
            assert r.flags & N.CT_SKIPPED_BUSY and r.mismatches == [0, 0, 0] and r.ms == [0, 0, 0], r
            (p,) = ctx.probe_health(min_gbs=1e-3)
            assert not p.flags & N.RES_COMPUTE
            (r,) = ctx.sfu_test(0, duration_ms=10, even_if_busy=True)
            assert not r.flags & N.CT_SKIPPED_BUSY and r.healthy and r.err == 0, r
    finally:
        if helper.poll() is None:
            helper.kill()
        helper.wait()


def test_daemon_sfu_test_at_start_logs_a_clean_result(short_dir):
    exe = os.path.join(ROOT, "k8s-device-plugin_b200", "b200dp_plugind")

    def lines(level):
        proc = subprocess.Popen([exe, "-backend=cuda:devices=0,bytes=67108864,calib=1", "-plugin_dir", short_dir,
                                 "-start_retry_wait=0.05", "-sfu_test_at_start=%d" % level, "-compute_test_ms=50"],
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
        assert log.index("sfu test ") < log.index("Failed to start plugin"), log[-3000:]
        return [ln for ln in log.splitlines() if ln.startswith("sfu test ")], log

    got, log = lines(1)
    assert len(got) == 1, log[-3000:]
    if "flags 0x1," in got[0]:
        got, log = lines(2)
        assert len(got) == 1, log[-3000:]
    assert ": Healthy, flags 0x" in got[0] and "mismatches 0/0/0, first bad SM -1" in got[0], log[-3000:]
