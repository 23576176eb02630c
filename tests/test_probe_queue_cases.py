"""The cases tests/test_gpu_probe_queue.py runs through hbm_probe_queue (tests/probe_cases.py with the queue kernel's
shape) reach what that test claims: every ring edge of the 6-stage pipeline, the queue's edges, every tail class, every
fault class and lane, and both deltas.  The properties are recomputed from the numbers (n_vec, grid, corrupted words),
not read from the case labels.  No GPU needed."""

import probe_cases as pc
from oracle import probe as oprobe
from probe_queue_kernels import QUEUE

def test_shape_matches_the_harness():
    import probe_queue_kernels
    assert probe_queue_kernels.variant() == QUEUE

def test_launch_shapes_reach_the_ring_and_queue_edges():
    """With one CTA the queue hands it every tile, so a grid-1 case with k tiles runs the ring exactly k deep: the
    cases must cover each count where the loader, storer and verifiers change shape (the empty-barrier wait starts at
    k = S, the parity flips every S tiles, the end-of-work slot lands in each position of the first two laps).  At
    larger grids, every CTA makes one claim past the last tile; the cases must include grids with fewer tiles than
    CTAs (CTAs whose first claim is already past the end), no tiles at all, and grids that do not divide the tiles."""
    c, s = QUEUE.vec_per_tile, QUEUE.stages
    cases = pc.cases(QUEUE)
    one_cta = {x.n_vec // c for x in cases if x.grid == 1}
    assert set(range(0, 3)) | {s - 1, s, s + 1, 2 * s - 1, 2 * s, 2 * s + 1} <= one_cta, sorted(one_cta)
    n_tiles = [(x.n_vec // c, x.grid) for x in cases]
    assert any(0 < t < g for t, g in n_tiles)                       # CTAs that get no tile
    assert any(t == 0 and g > 1 for t, g in n_tiles)                 # every claim is past the end
    assert any(t % g for t, g in n_tiles if t >= g > 1)              # uneven split
    assert any(t >= 2 * s * g for t, g in n_tiles if g > 1)          # several laps per CTA on a multi-CTA grid
    assert QUEUE.product_grid() in {g for _, g in n_tiles}
    assert {0, 1, 2, c - 1} <= {x.n_vec % c for x in cases if x.n_vec >= c}
    assert set(pc.SMALL_N_VEC) <= {x.n_vec for x in cases}
    assert max(x.n_vec for x in cases) * 16 <= 64 << 20

def test_faults_cover_every_class_and_lane():
    seen, lanes = set(), set()
    for x in pc.cases(QUEUE):
        seen.add(x.fault)
        src = x.src()
        cs, bad, first, _ = oprobe.probe_pass(src, x.seed, x.seed ^ x.delta)
        if x.fault == "clean":
            assert (bad, first, cs) == (0, oprobe.NO_BAD, oprobe.expected_checksum(x.n_words, x.seed))
        elif x.fault.startswith("lane"):
            assert bad == 1 and first == x.words[0] and x.words[0] % 4 == int(x.fault[4])
            lanes.add(x.words[0] % 4)
        elif x.fault == "pair":
            assert cs == oprobe.expected_checksum(x.n_words, x.seed) and bad == 2
        elif x.fault == "random":
            assert bad > 0.99 * x.n_words - 8
        else:
            assert bad == len(x.words) and first == x.words[0]
    assert seen == set(pc.FAULTS)
    assert lanes == {0, 1, 2, 3}

def test_every_case_runs_advancing_and_verify_only():
    by = {}
    for x in pc.cases(QUEUE):
        by.setdefault((x.name.rsplit(":", 1)[0], x.seed), []).append(x.delta)
    for (_, seed), deltas in by.items():
        assert sorted(deltas) == [0, seed ^ oprobe.next_seed(seed)]
