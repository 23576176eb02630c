"""Launch-shape and fault cases for the HBM probe kernels (pure Python; used by tests/test_gpu_kernels.py and checked
without a GPU by tests/test_probe_cases.py).

The kernels split a buffer of n_vec 16-byte vectors into full tiles (TMA variants) or chunks (register variants) of C
vectors, hand tile t to CTA t mod grid, and stream the remaining n_vec mod C vectors (the ragged tail) through a
grid-stride register loop.  A TMA CTA runs its tiles through a ring of S stages: the prologue loads min(k, S) tiles,
tile k-1+S is loaded after tile k is stored, and the mbarrier parity flips every S tiles.  The cases put every CTA at
the counts where that pipeline changes shape (k = 0, 1, 2, S-1, S, S+1, 2S-1, 2S, 2S+1), split tiles unevenly, give the
grid more CTAs than tiles, and add ragged tails, then corrupt the source in ways a per-vector or per-checksum shortcut
would miss.  Everything is derived from fixed seeds, so the cases are the same on every run."""
import zlib
from dataclasses import dataclass
from typing import Tuple

import numpy as np

from oracle import probe as oprobe

H100_SMS = 132


@dataclass(frozen=True)
class Variant:
    name: str
    vec_per_tile: int     # vectors per TMA tile or register-path chunk
    stages: int           # TMA ring depth, 0 for the register paths
    threads: int          # threads per CTA
    ctas_per_sm: int      # grid 0 launches SMs x this

    def product_grid(self, sms=H100_SMS):
        return sms * self.ctas_per_sm


# Mirrors the table in tests/native/probe_kernels.cu (tests/test_probe_cases.py checks that the two agree).
VARIANTS = (
    Variant("tma_4_1024_3", 1024, 3, 160, 2),
    Variant("r128_512_2", 1024, 0, 512, 2),
    Variant("tma_4_1024_3_h1", 1024, 3, 160, 2),
    Variant("tma_4_1024_3_h2", 1024, 3, 160, 2),
    Variant("tma_4_1024_3_h4", 1024, 3, 160, 2),
    Variant("tma_4_1024_3_h8", 1024, 3, 160, 2),
    Variant("tma_4_512_6", 512, 6, 160, 2),
    Variant("tma_2_1024_4", 1024, 4, 96, 2),
    Variant("tma_8_2048_3", 2048, 3, 288, 2),
    Variant("r256_256_1", 512, 0, 256, 2),
    Variant("r256_512_2", 2048, 0, 512, 2),
)

# fault classes, in the order they are handed out
FAULTS = ("clean", "lane0", "lane1", "lane2", "lane3", "multi", "boundary", "last_cta", "tail", "dense", "random", "pair")

SMALL_N_VEC = (0, 1, 2, 3)


def tile_counts(s):
    """Per-CTA tile counts where a ring of S stages changes shape (S = 0: register path, no ring)."""
    return tuple(sorted({k for k in (0, 1, 2, s - 1, s, s + 1, 2 * s - 1, 2 * s, 2 * s + 1) if k >= 0}))


def tails(c):
    return (0, 1, 2, c - 1)


def per_cta_tiles(n_vec, grid, c):
    """Full tiles (chunks) each CTA streams: tile t goes to CTA t mod grid."""
    n_tiles = n_vec // c
    return [(n_tiles - b + grid - 1) // grid if n_tiles > b else 0 for b in range(grid)]


@dataclass(frozen=True)
class Case:
    name: str
    n_vec: int
    grid: int
    fault: str                     # one of FAULTS
    words: Tuple[int, ...]         # corrupted word indices (ascending)
    masks: Tuple[int, ...]         # XOR mask of each corrupted word
    random_src: bool               # the whole source is random words (fault "random")
    seed: int
    delta: int                     # seed ^ next_seed (an advancing pass) or 0 (verify-only, as the P2P pass)

    @property
    def n_words(self):
        return 4 * self.n_vec

    def src(self):
        """The source buffer (uint32 words) this case feeds the kernel."""
        if self.random_src:
            buf = np.random.default_rng([self.seed, 0xA11]).integers(0, 1 << 32, self.n_words, dtype=np.uint32)
        else:
            buf = oprobe.pattern(self.n_words, self.seed)
        if self.words:
            buf[np.array(self.words, dtype=np.int64)] ^= np.array(self.masks, dtype=np.uint32)
        return buf


def _faults(kind, n_vec, grid, c, seed):
    """(words, masks, random_src) for fault class `kind`, or None when the shape has no room for it."""
    rng = np.random.default_rng([seed, zlib.crc32(kind.encode())])
    n_words = 4 * n_vec
    n_tiles = n_vec // c
    bit = lambda: 1 << int(rng.integers(0, 32))             # noqa: E731
    if kind == "clean":
        return (), (), False
    if kind == "random":
        return ((), (), True) if n_vec else None
    if kind.startswith("lane"):                              # one bad word, in lane x / y / z / w of one vector
        if not n_vec:
            return None
        v = int(rng.integers(0, n_vec))
        return (4 * v + int(kind[4]),), (bit(),), False
    if kind == "multi":                                      # several bad words in one vector, the first not in lane x
        if not n_vec:
            return None
        v = int(rng.integers(0, n_vec))
        lanes = (1, 3) if rng.integers(0, 2) else (1, 2, 3)
        return tuple(4 * v + ln for ln in lanes), tuple(bit() for _ in lanes), False
    if kind == "boundary":                                   # first and last word of a tile, first word after it
        if not n_tiles:
            return None
        t = int(rng.integers(0, n_tiles))
        ws = [4 * c * t, 4 * c * (t + 1) - 1]
        if 4 * c * (t + 1) < n_words:
            ws.append(4 * c * (t + 1))
        return tuple(ws), tuple(bit() for _ in ws), False
    if kind == "last_cta":                                   # only in the last CTA's last tile: min(first_bad) not in CTA 0
        k_last = per_cta_tiles(n_vec, grid, c)[-1]
        if grid < 2 or not k_last:
            return None
        t = grid - 1 + (k_last - 1) * grid
        ws = sorted(set(int(w) for w in 4 * c * t + rng.integers(0, 4 * c, 3)))
        return tuple(ws), tuple(bit() for _ in ws), False
    if kind == "tail":                                       # only past the last full tile
        lo = 4 * c * n_tiles
        if lo >= n_words:
            return None
        ws = sorted(set(int(w) for w in rng.integers(lo, n_words, 2)) | {n_words - 1})
        return tuple(ws), tuple(bit() for _ in ws), False
    if kind == "dense":                                      # a random 1 % of the words, any nonzero masks
        if not n_vec:
            return None
        m = max(1, n_words // 100)
        ws = np.sort(rng.choice(n_words, size=m, replace=False))
        masks = rng.integers(1, 1 << 32, m, dtype=np.uint64)
        return tuple(int(w) for w in ws), tuple(int(x) for x in masks), False
    if kind == "pair":                                       # bit b 0->1 in one word and 1->0 in another: sum unchanged
        if n_words < 2:
            return None
        pat = oprobe.pattern(n_words, seed)
        for _ in range(64):
            b = int(rng.integers(0, 32))
            bits = (pat >> np.uint32(b)) & np.uint32(1)
            zeros, ones = np.nonzero(bits == 0)[0], np.nonzero(bits == 1)[0]
            if zeros.size and ones.size:
                i, j = int(rng.choice(zeros)), int(rng.choice(ones))
                return tuple(sorted((i, j))), (1 << b, 1 << b), False
        return None
    raise ValueError(kind)


def shapes(v: Variant, product_grid: int):
    """(label, n_vec, grid) launch shapes for variant v."""
    c, s, g_p = v.vec_per_tile, v.stages, product_grid
    out = []
    tl = tails(c)
    i = 0
    # every CTA streams exactly k tiles; small grids keep the large k cheap
    for g in (1, 3, 7):
        for k in tile_counts(s):
            out.append(("even_g%d_k%d_t%d" % (g, k, tl[i % 4]), g * k * c + tl[i % 4], g))
            i += 1
    for k in sorted({1, 2, s, s + 1} - {0}):
        out.append(("even_gP_k%d_t%d" % (k, tl[i % 4]), g_p * k * c + tl[i % 4], g_p))
        i += 1
    # uneven: the first r CTAs stream one tile more
    for g, k, r in ((3, 1, 1), (7, max(s, 1), 3), (7, 2 * s + 1, 6), (g_p, 1, g_p // 2)):
        out.append(("uneven_g%d_k%d_r%d_t%d" % (g, k, r, tl[i % 4]), (g * k + r) * c + tl[i % 4], g))
        i += 1
    # more CTAs than tiles
    for g, n_tiles in ((7, 3), (g_p, 5), (g_p, g_p - 1)):
        out.append(("sparse_g%d_n%d_t%d" % (g, n_tiles, tl[i % 4]), n_tiles * c + tl[i % 4], g))
        i += 1
    # fewer vectors than one tile, down to nothing
    for n in SMALL_N_VEC:
        out.append(("small_gP_n%d" % n, n, g_p))
    out.append(("small_g1_n3", 3, 1))
    return out


def cases(v: Variant, product_grid: int = None):
    """Every case for variant v on a part whose product grid is `product_grid` (default: an H100 SXM's)."""
    g_p = product_grid or v.product_grid()
    rng = np.random.default_rng(zlib.crc32(v.name.encode()))
    out = []
    used = dict.fromkeys(FAULTS, 0)
    for i, (label, n_vec, grid) in enumerate(shapes(v, g_p)):
        seed = int(rng.integers(0, 1 << 32))
        # the least used fault class this shape has room for (ties: rotate through FAULTS)
        room = {}
        for step in range(len(FAULTS)):
            kind = FAULTS[(i + step) % len(FAULTS)]
            f = _faults(kind, n_vec, grid, v.vec_per_tile, seed)
            if f is not None and not any(used[k] <= used[kind] for k in room):
                room = {kind: f}
        (kind, (words, masks, random_src)), = room.items()
        used[kind] += 1
        for delta in (seed ^ oprobe.next_seed(seed), 0):
            out.append(Case("%s:%s:%s" % (label, kind, "adv" if delta else "verify"), n_vec, grid, kind, words, masks,
                            random_src, seed, delta))
    return out
