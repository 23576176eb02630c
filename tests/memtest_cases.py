"""Launch-shape and fault cases for the memory-test march hbm_march_tma (pure Python; used by
tests/test_gpu_memtest_cases.py and checked without a GPU by tests/test_memtest_cases_cpu.py).

Tile t of a march belongs to segment t / tiles_per_seg and goes to CTA t mod grid; each CTA streams its k tiles
through a ring of S = 3 stages, and the three modes take different paths through it (WRITE arms full[s] with a plain
arrive, READ refills a slot once its verifiers are done, READ_WRITE refills it once the store of the previous tile has
read it).  Every case runs all four elements, so every mode meets every shape:

- every CTA streaming exactly k tiles, for every k where the ring changes shape, at grids 1, 3 and 7, and k = 1..4 at
  the product grid (SMs x 2);
- uneven splits, and more CTAs than tiles (CTAs with no tile at all);
- one-tile segments, segments whose tile count is not a power of two, a last segment of one tile, and 256 segments
  (the whole segment table);
- segments that do not lie in memory in table order: the GPU test carves one allocation into slots and puts
  segment g in slot `slots[g]`.

Faults are memtest_faults.Fault cells: XOR flips after E0, E1 or E2, stuck-at and transition cells, in every lane, at
tile and segment edges, only in the last CTA's last tile, densely, as a checksum-preserving pair and in segments 128
and 255 of the full table.  The initial buffer (before E0) is SENTINEL, which decides what a transition cell holds
after E0.  Everything is derived from fixed seeds, so the cases are the same on every run."""
import zlib
from dataclasses import dataclass
from typing import Tuple

import numpy as np

import memtest_faults as mf
import probe_cases as pc

STAGES = 3                            # kTmaStages
TILE_WORDS = 4096                     # 16 KiB tiles (kTmaTileVec x 4)
H100_PRODUCT_GRID = 2 * pc.H100_SMS   # kTmaCtasPerSm x SMs of an H100 SXM
SENTINEL = 0xA5A5A5A5                 # every word of a case before E0 (its bits are 1,0,1,0,0,1,0,1 from bit 0)
MAX_CASE_BYTES = 64 << 20

# fault classes, in the order they are handed out; SEG_TABLE only goes to the 256-segment shapes
FAULTS = ("clean", "lane0", "lane1", "lane2", "lane3", "multi", "tile_edges", "segment_edges", "last_cta", "dense",
          "pair", "xor1", "xor2", "stuck0", "stuck1", "tf_up", "tf_down")
SEG_TABLE = "segments_128_255"


def per_cta_tiles(n_tiles, grid):
    return pc.per_cta_tiles(n_tiles, grid, 1)


def segment_tiles(n_tiles, tiles_per_seg):
    """Tiles of each segment: all but the last hold tiles_per_seg, the last the remainder."""
    full, rest = divmod(n_tiles, tiles_per_seg)
    return (tiles_per_seg,) * full + ((rest,) if rest else ())


@dataclass(frozen=True)
class Case:
    name: str
    seg_tiles: Tuple[int, ...]        # tiles of each segment, in table order
    grid: int
    slots: Tuple[int, ...]            # slot of segment g in the GPU test's allocation (a permutation)
    fault: str                        # one of FAULTS or SEG_TABLE
    faults: Tuple[mf.Fault, ...]      # ascending by word
    seed: int

    @property
    def seg_words(self):
        return [t * TILE_WORDS for t in self.seg_tiles]

    @property
    def n_tiles(self):
        return sum(self.seg_tiles)

    @property
    def n_words(self):
        return self.n_tiles * TILE_WORDS

    def march(self):
        return mf.march_faulty(self.seg_words, self.seed, SENTINEL, self.faults)


def shapes(g_p):
    """(label, n_tiles, grid, tiles_per_seg).  Labels name the product grid gP, so they do not depend on the part."""
    out = []
    cycle = (1, 3, 2, 5, 7, 6, 4)
    i = 0
    for g in (1, 3, 7):                                # every CTA streams exactly k tiles
        for k in pc.tile_counts(STAGES):
            if k:
                tps = cycle[i % len(cycle)]
                out.append(("even_g%d_k%d_s%d" % (g, k, tps), g * k, g, tps))
                i += 1
    for k, tps in ((1, 5), (2, 7), (3, 6), (4, 5)):    # at most 4 x 320 / 5 = 256 segments for up to 160 SMs
        out.append(("even_gP_k%d_s%d" % (k, tps), g_p * k, g_p, tps))
    # uneven: the first r CTAs stream one tile more
    for g, k, r, tps, label in ((3, 1, 1, 1, "r1"), (7, 3, 3, 5, "r3"), (7, 7, 6, 6, "r6"),
                                (g_p, 1, g_p // 2, 3, "rhalf")):
        out.append(("uneven_g%s_k%d_%s_s%d" % (g if g != g_p else "P", k, label, tps), g * k + r, g, tps))
    # more CTAs than tiles
    for g, n, tps, label in ((3, 2, 1, "n2"), (7, 3, 2, "n3"), (7, 6, 4, "n6"), (g_p, 5, 3, "n5"),
                             (g_p, g_p - 1, 7, "nPm1")):
        out.append(("sparse_g%s_%s_s%d" % (g if g != g_p else "P", label, tps), n, g, tps))
    # the whole segment table: 256 one-tile segments, and 255 three-tile segments and a one-tile one
    for n, tps in ((256, 1), (3 * 255 + 1, 3)):
        for g in (7, g_p):
            out.append(("table256_g%s_s%d" % (g if g != g_p else "P", tps), n, g, tps))
    return out


def _bit_where(rng, value, want):
    """A random bit position of `value` that is `want`."""
    return int(rng.choice([b for b in range(32) if (value >> b) & 1 == want]))


def _faults(kind, seg_tiles, grid, seed, pattern):
    """The faults of class `kind` (ascending by word), or None when the shape has no room for it."""
    rng = np.random.default_rng([seed, zlib.crc32(kind.encode())])
    seg_words = [t * TILE_WORDS for t in seg_tiles]
    starts = np.cumsum([0] + seg_words)
    n_words = int(starts[-1])
    n_tiles = n_words // TILE_WORDS
    bit = lambda: 1 << int(rng.integers(0, 32))                            # noqa: E731
    xor0 = lambda ws: tuple(mf.Fault(int(w), "xor@0", bit()) for w in ws)  # noqa: E731
    if kind == "clean":
        return ()
    if kind.startswith("lane"):                        # one bad word, in lane x / y / z / w of one vector
        return xor0([4 * int(rng.integers(0, n_words // 4)) + int(kind[4])])
    if kind == "multi":                                # several bad words in one vector, the first not in lane x
        v = int(rng.integers(0, n_words // 4))
        return xor0([4 * v + ln for ln in ((1, 3) if rng.integers(0, 2) else (1, 2, 3))])
    if kind == "tile_edges":                           # first and last word of a tile, first word after it
        t = int(rng.integers(0, n_tiles))
        return xor0([w for w in (TILE_WORDS * t, TILE_WORDS * (t + 1) - 1, TILE_WORDS * (t + 1)) if w < n_words])
    if kind == "segment_edges":                        # first and last word of a segment, first word of the next
        g = int(rng.integers(0, len(seg_words)))
        return xor0([w for w in (starts[g], starts[g + 1] - 1, starts[g + 1]) if w < n_words])
    if kind == "last_cta":                             # only in the last CTA's last tile: min(first_bad) not in CTA 0
        k_last = per_cta_tiles(n_tiles, grid)[-1]
        if grid < 2 or not k_last:
            return None
        t = grid - 1 + (k_last - 1) * grid
        return xor0(sorted(set(int(w) for w in TILE_WORDS * t + rng.integers(0, TILE_WORDS, 3))))
    if kind == "dense":                                # a random 1 % of the words, any model, any nonzero mask
        ws = np.sort(rng.choice(n_words, size=max(1, n_words // 100), replace=False))
        models = rng.integers(0, len(mf.MODELS), ws.size)
        masks = rng.integers(1, 1 << 32, ws.size, dtype=np.uint64)
        return tuple(mf.Fault(int(w), mf.MODELS[m], int(x)) for w, m, x in zip(ws, models, masks))
    if kind == "pair":                                 # bit b 0 -> 1 in one word and 1 -> 0 in another: sums unchanged
        b = int(rng.integers(0, 32))
        bits = (pattern >> np.uint32(b)) & np.uint32(1)
        i, j = int(rng.choice(np.flatnonzero(bits == 0))), int(rng.choice(np.flatnonzero(bits == 1)))
        return tuple(mf.Fault(w, "xor@0", 1 << b) for w in sorted((i, j)))
    if kind in ("xor1", "xor2"):                       # flips after E1 / E2: the earlier elements read a clean word
        ws = sorted(set(int(w) for w in rng.integers(0, n_words, 2)))
        return tuple(mf.Fault(w, "xor@" + kind[3], int(rng.integers(1, 1 << 32))) for w in ws)
    if kind in mf.CELL_MODELS:                         # one faulty bit per word, at every (pattern bit, sentinel bit)
        out, used = [], set()
        for p in (0, 1):
            for s in (0, 1):
                b = _bit_where(rng, SENTINEL, s)
                while True:
                    w = int(rng.integers(0, n_words))
                    if w not in used and (int(pattern[w]) >> b) & 1 == p:
                        break
                used.add(w)
                out.append(mf.Fault(w, kind, 1 << b))
        return tuple(sorted(out))
    if kind == SEG_TABLE:                              # the far end of the segment table, every cell model
        if len(seg_words) != 256:
            return None
        ws = (starts[128], starts[128] + int(rng.integers(1, seg_words[128])), starts[255], starts[255] + 1, n_words - 1)
        models = ("xor@0", "stuck0", "stuck1", "tf_up", "tf_down")
        return tuple(mf.Fault(int(w), m, bit()) for w, m in zip(ws, models))
    raise ValueError(kind)


def cases(product_grid=H100_PRODUCT_GRID):
    """Every case, on a part whose product grid is `product_grid` (default: an H100 SXM's)."""
    rng = np.random.default_rng(zlib.crc32(b"hbm_march_tma"))
    used = dict.fromkeys(FAULTS, 0)
    out = []
    for i, (label, n_tiles, grid, tps) in enumerate(shapes(product_grid)):
        seed = int(rng.integers(0, 1 << 32))
        seg_tiles = segment_tiles(n_tiles, tps)
        slots = tuple(int(x) for x in rng.permutation(len(seg_tiles)))
        if slots == tuple(sorted(slots)):
            slots = slots[::-1]
        pattern = mf.expected([t * TILE_WORDS for t in seg_tiles], seed)
        faults = _faults(SEG_TABLE, seg_tiles, grid, seed, pattern)
        if faults is not None:
            kind = SEG_TABLE
        else:
            # the least used fault class this shape has room for (ties: rotate through FAULTS)
            room = {}
            for step in range(len(FAULTS)):
                k = FAULTS[(i + step) % len(FAULTS)]
                f = _faults(k, seg_tiles, grid, seed, pattern)
                if f is not None and not any(used[x] <= used[k] for x in room):
                    room = {k: f}
            (kind, faults), = room.items()
            used[kind] += 1
        out.append(Case("%s:%s" % (label, kind), seg_tiles, grid, slots, kind, faults, seed))
    return out
