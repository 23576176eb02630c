"""The memory-test march cases (tests/memtest_cases.py) and the faulty-memory oracle (tests/memtest_faults.py), without a
GPU.  The properties are recomputed here from the numbers (segments, grid, faulty words, the oracle's results), not
read from the case labels.  The detection table is written out by hand: it is what the march claims, and the oracle
has to agree with it for every bit and lane."""
import numpy as np
import pytest

import memtest_cases as mc
import memtest_faults as mf
import memtest_oracle as mt
import probe_cases as pc
from oracle import probe as oprobe

TW = mc.TILE_WORDS
ONES = 0xFFFFFFFF


@pytest.fixture(scope="module")
def cases():
    return mc.cases()


class Result:
    """One case through the oracle, faulty and clean: the (checksum, mismatches, first_bad) of each element, and what
    each reading element read, summarised as its checksum and its wrong words.  E1 and E2 store what they read ^ ~0,
    so the words they read follow from the buffers they left."""

    def __init__(self, c):
        res = c.march()
        self.res = [r[:3] for r in res]
        self.clean = [r[:3] for r in mf.march_faulty(c.seg_words, c.seed, mc.SENTINEL)]
        pattern = mf.expected(c.seg_words, c.seed)
        self.read_sum, self.bad = {}, {}
        for k in (1, 2, 3):
            read = res[k][3] ^ np.uint32(ONES) if mt.MARCH[k][1] else res[k][3]
            self.read_sum[k] = oprobe.checksum(read)
            self.bad[k] = np.flatnonzero(read != pattern ^ np.uint32(mt.MARCH[k][2]))


@pytest.fixture(scope="module")
def results(cases):
    return {c.name: Result(c) for c in cases}


# ---- the fault models ------------------------------------------------------------------------------------------------
def test_cell_models_on_one_bit():
    """Each model on one bit for every (before, written) pair, and bits outside the mask untouched."""
    want = {  # (before, written) -> stored
        "stuck0": {(0, 0): 0, (0, 1): 0, (1, 0): 0, (1, 1): 0},
        "stuck1": {(0, 0): 1, (0, 1): 1, (1, 0): 1, (1, 1): 1},
        "tf_up": {(0, 0): 0, (0, 1): 0, (1, 0): 0, (1, 1): 1},
        "tf_down": {(0, 0): 0, (0, 1): 1, (1, 0): 1, (1, 1): 1},
    }
    for model, table in want.items():
        for b in (0, 13, 31):
            for (before, written), stored in table.items():
                for rest in (0, ONES):
                    bw = (rest & ~(1 << b) | before << b) & ONES
                    ww = (~rest & ~(1 << b) | written << b) & ONES
                    got = int(mf.cell_after_write(model, 1 << b, 1, bw, ww))
                    assert got == (ww & ~(1 << b) | stored << b) & ONES, (model, b, before, written, rest)
    for k in (0, 1, 2):
        for elem in (0, 1, 2):
            got = int(mf.cell_after_write("xor@%d" % k, 0x80000001, elem, 0x1234, 0x5678))
            assert got == (0x5678 ^ 0x80000001 if elem == k else 0x5678)


def test_xor_after_e0_is_the_healthy_oracles_fault():
    """xor@0 reproduces memtest_oracle.march exactly: every result and every buffer, from any initial buffer."""
    words = [3 * TW, 3 * TW, TW]
    faults = [(0, 0x1), (3 * TW - 1, 0x80000000), (3 * TW, ONES), (5 * TW + 2, 0x00F0F000), (7 * TW - 1, 0x40)]
    for initial in (0, mc.SENTINEL, np.arange(7 * TW, dtype=np.uint32)):
        got = mf.march_faulty(words, 0x5EED1234, initial, [mf.Fault(w, "xor@0", m) for w, m in faults])
        want = mt.march(words, 0x5EED1234, faults)
        for g, w in zip(got, want):
            assert g[:3] == w[:3] and np.array_equal(g[3], w[3])


def test_pattern_sum_across_the_wrap():
    for base, n, chunk in ((0, 3 * TW, 1 << 24), ((1 << 32) - 5000, 9000, 1 << 24), ((1 << 32) - 5000, 9000, 4096),
                           ((1 << 32) - 4096, 4096, 4096), (5 << 32, 100, 7)):
        assert mf.pattern_sum(base, n, 0xC0FFEE, chunk) == mt.range_checksum(base, n, 0xC0FFEE), (base, n, chunk)


# ---- the detection table ---------------------------------------------------------------------------------------------
# (model, pattern bit p, sentinel bit s before E0, counted in [E1, E2, E3]); None = either value
DETECTION = [
    ("stuck0", 1, None, [1, 0, 1]),     # stuck-at-v, p != v
    ("stuck1", 0, None, [1, 0, 1]),
    ("stuck0", 0, None, [0, 1, 0]),     # stuck-at-v, p == v
    ("stuck1", 1, None, [0, 1, 0]),
    ("tf_up", 0, None, [0, 1, 0]),
    ("tf_up", 1, 1, [0, 0, 1]),
    ("tf_up", 1, 0, [1, 0, 1]),
    ("tf_down", 1, None, [0, 1, 0]),
    ("tf_down", 0, 0, [0, 0, 1]),
    ("tf_down", 0, 1, [1, 0, 1]),
    ("xor@0", None, None, [1, 1, 1]),
    ("xor@1", None, None, [0, 1, 1]),
    ("xor@2", None, None, [0, 0, 1]),
]


def test_detection_table_has_no_blind_row():
    assert all(any(counts) for _, _, _, counts in DETECTION)
    covered = {(m, p, s) for m, p0, s0, _ in DETECTION for p in ((0, 1) if p0 is None else (p0,))
               for s in ((0, 1) if s0 is None else (s0,))}
    assert covered == {(m, p, s) for m in mf.MODELS for p in (0, 1) for s in (0, 1)}


@pytest.mark.parametrize("lane", range(4))
def test_one_faulty_bit_is_caught_where_the_table_says(lane):
    """One tile, one faulty bit: for every bit 0-31 in this lane, every model and every (p, s), the reading elements
    that count it are the table's, and each of them reports that word as the first bad one.  Bits 0 and 1 of a lane
    are the same in every vector under one seed (K is odd), so the seed is chosen to give the word its pattern bit."""
    pattern = mf.expected([TW], 0x3C5A0F11)
    for b in range(32):
        w = 4 * 17 * b + lane
        for model, p0, s0, counts in DETECTION:
            for p in ((0, 1) if p0 is None else (p0,)):
                seed = 0x3C5A0F11 ^ ((int(pattern[w]) >> b & 1 ^ p) << b)
                assert int(mf.expected([TW], seed)[w]) >> b & 1 == p
                for s in ((0, 1) if s0 is None else (s0,)):
                    initial = np.full(TW, mc.SENTINEL, dtype=np.uint32)
                    initial[w] = initial[w] & ~np.uint32(1 << b) | np.uint32(s << b)
                    res = mf.march_faulty([TW], seed, initial, [mf.Fault(w, model, 1 << b)])
                    assert res[0][:3] == (0, 0, mt.NO_BAD)
                    got = [res[k][1] for k in (1, 2, 3)]
                    assert got == counts, (model, b, lane, p, s, got)
                    assert all(res[k][2] == (w if res[k][1] else mt.NO_BAD) for k in (1, 2, 3))


# ---- the cases -------------------------------------------------------------------------------------------------------
def test_launch_shapes_cover_the_ring_edges(cases):
    g_p = mc.H100_PRODUCT_GRID
    even, seen, uneven, sparse = {}, {}, set(), set()
    for c in cases:
        counts = mc.per_cta_tiles(c.n_tiles, c.grid)
        assert sum(counts) == c.n_tiles
        seen.setdefault(c.grid, set()).update(counts)
        if len(set(counts)) == 1:
            even.setdefault(c.grid, set()).add(counts[0])
        else:
            k = min(counts)
            r = counts.count(k + 1)
            assert counts == [k + 1] * r + [k] * (c.grid - r)
            if k >= 1:
                uneven.add(c.grid)
        if c.n_tiles < c.grid:
            sparse.add(c.grid)
    assert pc.tile_counts(mc.STAGES) == (0, 1, 2, 3, 4, 5, 6, 7)
    for g in (1, 3, 7):
        assert set(range(1, 2 * mc.STAGES + 2)) <= even[g], (g, sorted(even[g]))
    # a march has at least one tile, so grid 1 never has an idle CTA; grids 3 and 7 do
    assert set(pc.tile_counts(mc.STAGES)) - {0} <= seen[1]
    assert set(pc.tile_counts(mc.STAGES)) <= seen[3] and set(pc.tile_counts(mc.STAGES)) <= seen[7]
    assert {1, 2, 3, 4} <= even[g_p]
    assert {3, 7, g_p} <= uneven and {3, 7, g_p} <= sparse


def test_segment_tables(cases):
    """Every table is one the harness launches, and together they reach its edges."""
    layouts = set()
    for c in cases:
        t = c.seg_tiles
        assert 1 <= len(t) <= 256 and all(x == t[0] for x in t[:-1]) and 1 <= t[-1] <= t[0]
        assert c.n_words * 4 <= mc.MAX_CASE_BYTES
        assert sorted(c.slots) == list(range(len(t)))
        if len(t) > 1:
            assert list(c.slots) != sorted(c.slots), c.name      # not in address order
            layouts.add("multi")
        if len(t) > 1 and set(t) == {1}:
            layouts.add("one_tile_segments")
        if t[0] & (t[0] - 1):
            layouts.add("not_power_of_two")
        if len(t) > 1 and t[0] > 1 and t[-1] == 1:
            layouts.add("last_of_one_tile")
        if len(t) == 256 and set(t) == {1}:
            layouts.add("256x1")
        if len(t) == 256 and t[0] == 3 and t[-1] == 1:
            layouts.add("255x3+1")
    assert layouts == {"multi", "one_tile_segments", "not_power_of_two", "last_of_one_tile", "256x1", "255x3+1"}


def test_cases_do_not_depend_on_the_parts_sm_count():
    """The GPU test finds cases by name on whatever part it runs: the names are the same, and the tables still fit."""
    names = [c.name for c in mc.cases()]
    for sms in (114, 132, 144):
        other = mc.cases(2 * sms)
        assert [c.name for c in other] == names
        assert all(len(c.seg_tiles) <= 256 and c.n_words * 4 <= mc.MAX_CASE_BYTES for c in other)


def test_every_fault_is_caught_and_nothing_else(cases, results):
    """Per word: every faulty word is counted by at least one reading element, no other word is, and each element's
    count, first bad word and checksum agree with the words it read.  The faults change the result."""
    for c in cases:
        r = results[c.name]
        flagged = set()
        for k in (1, 2, 3):
            bad = r.bad[k]
            assert r.res[k] == (r.read_sum[k], bad.size, int(bad[0]) if bad.size else mt.NO_BAD), (c.name, k)
            flagged |= set(bad.tolist())
        assert flagged == {f.word for f in c.faults}, c.name
        assert r.res[0] == r.clean[0] == (0, 0, mt.NO_BAD)
        assert all(r.clean[k][1] == 0 and r.clean[k][0] == mt.expected_checksum(c.seg_words, c.seed, mt.MARCH[k][2])
                   for k in (1, 2, 3))
        if c.faults:
            assert any(r.res[k] != r.clean[k] for k in (1, 2, 3)), c.name


def test_faults_cover_every_class_lane_and_cell(cases, results):
    classes, lanes, cells = set(), set(), set()
    for c in cases:
        res, clean = results[c.name].res, results[c.name].clean
        ws = np.array([f.word for f in c.faults], dtype=np.int64)
        models = {f.model for f in c.faults}
        starts = np.cumsum([0] + c.seg_words)
        seg = np.searchsorted(starts, ws, side="right") - 1
        assert list(ws) == sorted(set(ws.tolist())) and all(f.mask for f in c.faults)
        classes.add(c.fault)
        pattern = mf.expected(c.seg_words, c.seed)
        lanes |= set((ws % 4).tolist())
        for f in c.faults:
            if f.model in mf.CELL_MODELS and f.mask & (f.mask - 1) == 0:
                b = f.mask.bit_length() - 1
                cells.add((f.model, int(pattern[f.word]) >> b & 1, mc.SENTINEL >> b & 1))
        mm = [res[k][1] for k in (1, 2, 3)]
        if not c.faults:
            assert c.fault == "clean"
        elif c.fault.startswith("lane"):
            assert len(ws) == 1 and ws[0] % 4 == int(c.fault[4]) and models == {"xor@0"} and mm == [1, 1, 1]
        elif c.fault == "multi":          # the first bad lane of the vector is not lane x
            assert len(ws) >= 2 and len(set(ws // 4)) == 1 and ws[0] % 4 != 0 and res[1][2] == ws[0]
        elif c.fault == "tile_edges":
            t = ws[0] // TW
            assert ws[0] == t * TW and ws[1] == (t + 1) * TW - 1 and (len(ws) == 2) == (ws[1] + 1 == c.n_words)
        elif c.fault == "segment_edges":
            assert ws[0] == starts[seg[0]] and ws[1] == starts[seg[0] + 1] - 1
        elif c.fault == "last_cta":       # every fault in CTA grid-1's last tile, so min(first_bad) is not in CTA 0
            k_last = mc.per_cta_tiles(c.n_tiles, c.grid)[-1]
            assert c.grid >= 2 and set((ws // TW).tolist()) == {c.grid - 1 + (k_last - 1) * c.grid}
            assert (res[1][2] // TW) % c.grid == c.grid - 1
        elif c.fault == "dense":
            assert len(ws) == c.n_words // 100 and models == set(mf.MODELS)
        elif c.fault == "pair":           # only the mismatch counts can fail this buffer
            assert models == {"xor@0"} and len(ws) == 2 and mm == [2, 2, 2]
            assert all(res[k][0] == clean[k][0] for k in (1, 2, 3))
        elif c.fault in ("xor1", "xor2"):  # E1..Ek read a clean buffer, every element after the flip sees it
            e = int(c.fault[3])
            assert models == {"xor@%d" % e} and all(m == 0 for m in mm[:e]) and all(mm[e:])
        elif c.fault in mf.CELL_MODELS:
            assert models == {c.fault} and len(ws) == 4
        elif c.fault == mc.SEG_TABLE:
            assert len(c.seg_words) == 256 and set(seg.tolist()) == {128, 255} and models >= set(mf.CELL_MODELS)
        else:
            raise AssertionError(c.fault)
    assert classes == set(mc.FAULTS) | {mc.SEG_TABLE}
    assert lanes == {0, 1, 2, 3}
    assert cells == {(m, p, s) for m in mf.CELL_MODELS for p in (0, 1) for s in (0, 1)}


def test_cases_are_deterministic(cases):
    again = mc.cases()
    assert again == cases
    assert len({c.name for c in cases}) == len(cases)
