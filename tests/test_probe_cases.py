"""The probe kernel cases (tests/probe_cases.py) cover what tests/test_gpu_kernels.py claims to test: every per-CTA
tile count at the TMA ring's edges, uneven splits, every tail class, every fault class and lane, and both deltas.  The
properties are recomputed here from the numbers (n_vec, grid, corrupted words), not read from the case labels.
No GPU needed."""
import numpy as np
import pytest

import probe_cases as pc
from oracle import probe as oprobe


def test_variant_table_matches_the_harness():
    import probe_kernels
    assert probe_kernels.variants() == list(pc.VARIANTS)


def test_required_tile_counts():
    assert pc.tile_counts(3) == (0, 1, 2, 3, 4, 5, 6, 7)
    assert pc.tile_counts(6) == (0, 1, 2, 5, 6, 7, 11, 12, 13)
    assert pc.tile_counts(0) == (0, 1, 2)


@pytest.mark.parametrize("v", pc.VARIANTS, ids=lambda v: v.name)
def test_launch_shapes_cover_the_pipeline_edges(v):
    c, s, g_p = v.vec_per_tile, v.stages, v.product_grid()
    cases = pc.cases(v)
    even = {}
    uneven = False
    sparse = False
    for x in cases:
        counts = pc.per_cta_tiles(x.n_vec, x.grid, c)
        n_tiles = x.n_vec // c
        if len(set(counts)) == 1:
            even.setdefault(x.grid, set()).add(counts[0])
        else:
            k = min(counts)
            r = counts.count(k + 1)
            assert counts == [k + 1] * r + [k] * (x.grid - r)
            uneven |= k >= 1
        sparse |= 0 < n_tiles < x.grid
    for g in (1, 3, 7):
        assert set(pc.tile_counts(s)) <= even[g], (g, sorted(even[g]))
    assert {1, 2} <= even[g_p]
    assert uneven and sparse
    assert {1, 3, 7, g_p} <= {x.grid for x in cases}
    assert {0, 1, 2, c - 1} <= {x.n_vec % c for x in cases if x.n_vec >= c}
    assert set(pc.SMALL_N_VEC) <= {x.n_vec for x in cases}
    assert max(x.n_vec for x in cases) * 16 <= 64 << 20


@pytest.mark.parametrize("v", pc.VARIANTS, ids=lambda v: v.name)
def test_faults_cover_every_class_and_lane(v):
    c = v.vec_per_tile
    seen = set()
    lanes = set()
    for x in pc.cases(v):
        seen.add(x.fault)
        src = x.src()
        assert src.dtype == np.uint32 and src.size == x.n_words
        cs, bad, first, _ = oprobe.probe_pass(src, x.seed, x.seed ^ x.delta)
        want_cs = oprobe.expected_checksum(x.n_words, x.seed)
        ws = np.array(x.words, dtype=np.int64)
        assert list(x.words) == sorted(set(x.words)) and all(m for m in x.masks)
        if x.fault == "clean":
            assert (bad, first, cs) == (0, oprobe.NO_BAD, want_cs)
        elif x.fault.startswith("lane"):
            assert len(ws) == 1 and bad == 1 and first == ws[0] and ws[0] % 4 == int(x.fault[4])
            lanes.add(int(ws[0] % 4))
        elif x.fault == "multi":      # the first bad lane of the vector is not its last one
            assert len(ws) >= 2 and len(set(ws // 4)) == 1 and bad == len(ws) and first == ws[0] and ws[0] % 4 != 0
        elif x.fault == "boundary":
            assert any(w % (4 * c) == 0 for w in ws) and any(w % (4 * c) == 4 * c - 1 for w in ws)
            assert bad == len(ws)
        elif x.fault == "last_cta":   # every fault in CTA grid-1's last tile, so min(first_bad) is not in CTA 0
            k_last = pc.per_cta_tiles(x.n_vec, x.grid, c)[-1]
            assert x.grid >= 2 and set(ws // (4 * c)) == {x.grid - 1 + (k_last - 1) * x.grid}
            assert (first // (4 * c)) % x.grid == x.grid - 1 and bad == len(ws)
        elif x.fault == "tail":
            assert x.n_vec % c and (ws >= 4 * c * (x.n_vec // c)).all() and ws[-1] == x.n_words - 1
        elif x.fault == "dense":
            assert len(ws) == max(1, x.n_words // 100) and bad == len(ws)
        elif x.fault == "random":
            assert x.random_src and bad > 0.99 * x.n_words - 8
        elif x.fault == "pair":       # only the mismatch count can fail this buffer
            assert cs == want_cs and bad == 2 and first == ws[0]
        else:
            raise AssertionError(x.fault)
    assert seen == set(pc.FAULTS)
    assert lanes == {0, 1, 2, 3}


@pytest.mark.parametrize("v", pc.VARIANTS, ids=lambda v: v.name)
def test_every_case_runs_advancing_and_verify_only(v):
    by = {}
    for x in pc.cases(v):
        by.setdefault((x.name.rsplit(":", 1)[0], x.n_vec, x.grid, x.words, x.seed), []).append(x.delta)
    for key, deltas in by.items():
        seed = key[-1]
        assert sorted(deltas) == [0, seed ^ oprobe.next_seed(seed)] and deltas[0] != 0, key


@pytest.mark.parametrize("v", pc.VARIANTS, ids=lambda v: v.name)
def test_cases_are_deterministic(v):
    a, b = pc.cases(v), pc.cases(v)
    assert a == b
    assert all(np.array_equal(x.src(), y.src()) for x, y in zip(a, b) if x.n_vec < 4096)
    assert len({x.name for x in a}) == len(a)
