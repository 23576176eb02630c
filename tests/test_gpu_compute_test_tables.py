"""The tensor-core self-test kernel (tc_selftest.cuh) on a real H100, on inputs the generator's fixed seeds never reach.
Every fault goes in through the tables the kernel reads -- operand images and per-thread check values -- so the path
under test is the product's own: operand bytes, tensor cores, fold, CTA-wide compare, record.
The inputs are in tests/compute_test_cases.py; tests/test_compute_test_tables_cpu.py checks what they reach.

- No false alarm: 256 seeds per format through the product's own table builder, every CTA of a full grid; the raw
  accumulators at the scanned edge seeds and on crafted tiles (every element at the bound, a late +-1 addend in every K
  step, exact zeros by cancellation) equal the oracle bit for bit.
- Every wrong product is caught: a wrong check value in each of the 128 threads (tile t mod 8), a wrong operand element
  in each warp's rows, in result columns 0 and 127 and in the first and last K step, a one-unit change of a result near
  2^24, and two wrong tiles.  Each is counted in every repetition of every round by every CTA of the grid.
- The harness refuses malformed input without launching.

Each launch runs for at most 5 ms."""
import ctypes as C
import os

import numpy as np
import pytest

import compute_test_cases as cc
import compute_test_oracle as ct
import compute_test_tables as tb
from test_gpu_compute_test import MS, CtRecord, Harness

pytestmark = pytest.mark.gpu

LIB_PATH = os.path.join(os.path.dirname(os.path.abspath(__file__)), "native", "libcompute_test_tables_test.so")
FMT_IDS = [ct.NAMES[f] for f in ct.FORMATS]
SEQ = 9                                 # ck_run_tables' launch sequence number
CK_E_FMT, CK_E_NOSPC, CK_E_SIZE, CK_E_GRID, CK_E_DUMP = -1, -2, -3, -4, -5
RUN_MS = 5                              # long enough for every CTA to run several rounds


class TablesHarness(Harness):
    """Harness's methods (ck_run, ck_dump, ...) on libcompute_test_tables_test.so, which holds those entry points as
    they are plus ck_run_tables."""

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
        L.ck_run_tables.argtypes = [C.c_void_p, C.c_int, C.c_int, C.c_void_p, C.c_uint64, C.c_void_p, C.c_int,
                                         C.c_uint64, C.POINTER(CtRecord), C.c_int, C.POINTER(C.c_int),
                                         C.POINTER(C.c_float), C.c_void_p]

    def run_tables_rc(self, fmt, images, checks, grid, duration_ms=0, dump=False, image_bytes=None, cap=None,
                      dump_out=True):
        """(return code, records, dump or None): ck_run_tables as it is, for the refusal tests."""
        images = np.ascontiguousarray(images, dtype=np.uint8)
        checks = np.ascontiguousarray(checks, dtype=np.uint32)
        cap = max(grid, 1) if cap is None else cap
        recs = (CtRecord * cap)()
        n, ms = C.c_int(), C.c_float()
        out = np.full(ct.TILES * ct.THREADS * ct.ACC, 0xFFFFFFFF, np.uint32) if dump and dump_out else None
        rc = self.L.ck_run_tables(self.h, fmt, int(dump), images.ctypes.data,
                                  images.nbytes if image_bytes is None else image_bytes, checks.ctypes.data, grid,
                                  int(duration_ms * MS), recs, cap, C.byref(n), C.byref(ms),
                                  None if out is None else out.ctypes.data)
        return rc, list(recs[:n.value]) if rc == 0 else [], None if out is None else out.reshape(ct.TILES, ct.THREADS, ct.ACC)

    def run_tables(self, fmt, images, checks, grid, duration_ms=0, dump=False):
        rc, recs, out = self.run_tables_rc(fmt, images, checks, grid, duration_ms, dump)
        self._check(rc, "ck_run_tables")
        return recs, out


@pytest.fixture(scope="module")
def H():
    if not os.path.exists(LIB_PATH):
        pytest.skip("run __graft_entry__.build() first")
    h = TablesHarness(0)
    yield h
    h.close()


def _rec(r):
    return dict(smid=r.smid, seq=r.seq, rounds=r.rounds, comparisons=r.comparisons, mismatches=r.mismatches,
                first_bad_tile=r.first_bad_tile, first_bad_rep=r.first_bad_rep)


def _clean(r, seq):
    return (r.seq == seq and r.rounds >= 1 and r.comparisons == r.rounds * ct.TILES * ct.REPS and r.mismatches == 0
            and (r.first_bad_tile, r.first_bad_rep) == (-1, -1))


# ---- no false alarm ---------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("fmt", ct.FORMATS, ids=FMT_IDS)
def test_seed_sweep_raises_no_false_alarm(H, fmt):
    """The product's table builder (ck_run), a full grid, one round per CTA: every record complete, no mismatch."""
    grid = H.sms * H.occupancy(fmt)
    bad = []
    for seed in cc.sweep_seeds(fmt):
        recs, _ = H.run(fmt, seed, 0)
        assert len(recs) == grid
        wrong = [_rec(r) for r in recs if not _clean(r, 7)]
        if wrong:
            bad.append((seed, len(wrong), wrong[0]))
    assert not bad, bad[:8]


EDGE_DUMPS = [(f, s) for f in ct.FORMATS for s in cc.edge_seeds(f)]


def _assert_dump_matches(got, rec, seq, named):
    """DUMP accumulators `got` (TILES x THREADS x ACC) equal the fragments of each (name, D bits) in `named`, bit for
    bit, and the launch's one CTA compared one round with no mismatch."""
    bad = []
    for t, (name, d) in enumerate(named):
        want = ct.fragments(d)
        if not np.array_equal(got[t], want):
            th, j = np.argwhere(got[t] != want)[0]
            bad.append("tile %d (%s): %d words differ; first thread %d reg %d got 0x%08x want 0x%08x"
                       % (t, name, int((got[t] != want).sum()), th, j, got[t][th, j], want[th, j]))
    assert not bad, "\n".join(bad)
    assert (rec.seq, rec.rounds, rec.comparisons, rec.mismatches) == (seq, 1, ct.TILES * ct.REPS, 0), _rec(rec)
    assert (rec.first_bad_tile, rec.first_bad_rep) == (-1, -1)


@pytest.mark.parametrize("fmt,seed", EDGE_DUMPS, ids=["%s-%d" % (ct.NAMES[f], s) for f, s in EDGE_DUMPS])
def test_dump_matches_the_oracle_at_the_edge_seeds(H, fmt, seed):
    """The four BF16 scale-exponent corners and the first seed with an exact-zero result in each format."""
    got, rec = H.dump(fmt, seed)
    _assert_dump_matches(got, rec, 1, [("seed %d" % seed, ct.tile(seed, fmt, t)[4]) for t in range(ct.TILES)])


@pytest.mark.parametrize("fmt", ct.FORMATS, ids=FMT_IDS)
def test_crafted_tiles_match_the_oracle_bit_for_bit(H, fmt):
    named = cc.crafted_tiles(fmt)
    images, checks = tb.tables(fmt, [t for _, t in named])
    (rec,), got = H.run_tables(fmt, images, checks, 1, dump=True)
    _assert_dump_matches(got, rec, SEQ, [(name, tb.reference(fmt, *tile)) for name, tile in named])
    # and the product instantiation agrees on every CTA of a full grid
    recs, _ = H.run_tables(fmt, images, checks, H.sms * H.occupancy(fmt))
    wrong = [_rec(r) for r in recs if not _clean(r, SEQ)]
    assert not wrong, wrong[:4]


# ---- every wrong product caught ---------------------------------------------------------------------------------------
@pytest.mark.parametrize("fmt", ct.FORMATS, ids=FMT_IDS)
def test_a_wrong_check_value_is_caught_in_every_thread_and_tile(H, fmt):
    """One CTA, one round: thread t's check value of tile t mod 8 with bit t mod 32 flipped is counted in every
    repetition of that tile and in no other comparison."""
    images, checks = tb.tables(fmt, cc.generator_tiles(fmt))
    bad = []
    for tile, t, mask in cc.check_flips():
        c = checks.copy()
        c[tile, t] ^= np.uint32(mask)
        (r,), _ = H.run_tables(fmt, images, c, 1)
        got = (r.seq, r.rounds, r.comparisons, r.mismatches, r.first_bad_tile, r.first_bad_rep)
        if got != (SEQ, 1, ct.TILES * ct.REPS, ct.REPS, tile, 0):
            bad.append((t, got))
    assert not bad, bad[:8]


def _assert_every_cta_counts_every_repetition(H, fmt, images, checks, bad_tiles):
    """The product on a full grid for RUN_MS: every CTA runs >= 2 rounds and counts every repetition of every bad tile
    in every round, first at the lowest bad tile's repetition 0."""
    grid = H.sms * H.occupancy(fmt)
    recs, _ = H.run_tables(fmt, images, checks, grid, RUN_MS)
    assert len(recs) == grid
    wrong = []
    for r in recs:
        ok = (r.seq == SEQ and r.rounds >= 2 and r.comparisons == r.rounds * ct.TILES * ct.REPS
              and r.mismatches == r.rounds * len(bad_tiles) * ct.REPS
              and (r.first_bad_tile, r.first_bad_rep) == (min(bad_tiles), 0))
        if not ok:
            wrong.append(_rec(r))
    assert not wrong, (len(wrong), wrong[:4])


OPERAND_CASES = [(f, i) for f in ct.FORMATS for i in range(len(cc.operand_plan(f)))]


def _operand_id(f, i):
    tile, op, row, k = cc.operand_plan(f)[i]
    return "%s-%s%d-k%d-tile%d" % (ct.NAMES[f], "AB"[op], row, k, tile)


@pytest.mark.parametrize("fmt,i", OPERAND_CASES, ids=[_operand_id(f, i) for f, i in OPERAND_CASES])
def test_a_wrong_operand_is_caught_by_every_cta_in_every_repetition(H, fmt, i):
    plan = cc.operand_plan(fmt)[i]
    clean = cc.generator_tiles(fmt)
    _, checks = tb.tables(fmt, clean)
    images, _ = tb.tables(fmt, cc.corrupt_operands(fmt, clean, [plan]))
    _assert_every_cta_counts_every_repetition(H, fmt, images, checks, [plan[0]])


ONE_UNIT_CASES = [(f, c) for f in ct.FORMATS for c in cc.one_unit_cases(f)]


@pytest.mark.parametrize("fmt,case", ONE_UNIT_CASES,
                         ids=["%s-%+d" % (ct.NAMES[f], cc.late_cases(f)[c][1]) for f, c in ONE_UNIT_CASES])
def test_a_one_unit_error_near_the_top_of_the_range_is_caught(H, fmt, case):
    """The late-addend tile with the partner of one +-1 product (last k of the last K step) set to 0: for BF16 the
    result moves by one ulp at >= 2^23.9."""
    crafted = [t for _, t in cc.crafted_tiles(fmt)]
    _, checks = tb.tables(fmt, crafted)
    images, _ = tb.tables(fmt, cc.one_unit_corruption(fmt, crafted, case))
    _assert_every_cta_counts_every_repetition(H, fmt, images, checks, [cc.LATE_TILE])


@pytest.mark.parametrize("fmt", ct.FORMATS, ids=FMT_IDS)
def test_two_wrong_tiles_are_both_counted(H, fmt):
    clean = cc.generator_tiles(fmt)
    _, checks = tb.tables(fmt, clean)
    images, _ = tb.tables(fmt, cc.corrupt_operands(fmt, clean, cc.TWO_TILE_PLAN))
    _assert_every_cta_counts_every_repetition(H, fmt, images, checks, [t for t, *_ in cc.TWO_TILE_PLAN])


# ---- the harness ------------------------------------------------------------------------------------------------------
def test_harness_refuses_bad_input(H):
    fmt = ct.INT8
    images, checks = tb.tables(fmt, cc.generator_tiles(fmt))
    full = H.sms * H.occupancy(fmt)
    refusals = [
        ("format -1", dict(fmt=-1), CK_E_FMT),
        ("format 3", dict(fmt=ct.FORMATS[-1] + 1), CK_E_FMT),
        ("image one byte short", dict(image_bytes=images.nbytes - 1), CK_E_SIZE),
        ("image one byte long", dict(image_bytes=images.nbytes + 1), CK_E_SIZE),
        ("images of another format", dict(image_bytes=ct.TILES * tb.SMEM[ct.BF16]), CK_E_SIZE),
        ("grid 0", dict(grid=0), CK_E_GRID),
        ("grid -1", dict(grid=-1), CK_E_GRID),
        ("grid above the resident CTAs", dict(grid=full + 1, cap=full + 1), CK_E_GRID),
        ("records do not fit", dict(grid=2, cap=1), CK_E_NOSPC),
        ("DUMP without a buffer", dict(dump=True, dump_out=False), CK_E_DUMP),
    ]
    for what, kw, code in refusals:
        args = dict(fmt=fmt, images=images, checks=checks, grid=1)
        args.update(kw)
        rc, recs, _ = H.run_tables_rc(**args)
        assert (rc, recs) == (code, []), what
    # and the same tables run when nothing is wrong with the call
    recs, _ = H.run_tables(fmt, images, checks, full)
    assert len(recs) == full and all(_clean(r, SEQ) for r in recs)
