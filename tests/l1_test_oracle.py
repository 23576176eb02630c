"""Independent restatement of the L1 self-test's host reference (csrc/l1_test_math.hpp), from the layout the kernel
comment states, the CUDA programming guide's texture-fetching formulas and the PTX ISA's tld4, and fault models of the
L1TEX unit and the constant cache.

- table(seed, fmt, tile):            a tile's four table words
- results(seed, fmt, tile, fault):   every thread's result words, [128, W] (L1_DATA: one block, line keys removed, even
                                     repetition)
- checks(seed, fmt, tile, fault):    every thread's check value (L1_DATA: the even and odd block folds of CTA 0 at K = 1)
- data_reads(seed, tile, K, c):      L1_DATA's raw values in DUMP order
- tex_addr(mode, x, m, n):           the texel a point-sampled normalized fetch resolves to (None: the border colour)

The fault models (FAULTS[fmt]) change what a faulty unit would return; VISIBLE[fmt][fault] names the tiles where the
model must change a check."""
import math

import numpy as np

THREADS, TILES = 128, 8
DATA, TEX, CONST = 0, 1, 2
M32 = 0xFFFFFFFF
BLOCK, LINE = 512, 32
TEX_W, TEX_H = 64, 128
TEXELS = TEX_W * TEX_H
STEPS = TEXELS // THREADS
BANK, WIN = 8192, 2048
WRAP, MIRROR, CLAMP, BORDER = 0, 1, 2, 3
LINE_MUL = 0x9E3779B9
PAT_MUL = 2654435761
FOLD_MUL, FOLD_ROT, FOLD_INIT = 2654435761, 13, (0x9E3779B1, 0x85EBCA77, 0xC2B2AE3D, 0x27D4EB2F)


def ct_mix(x):
    x &= M32
    x ^= x >> 16
    x = (x * 0x7FEB352D) & M32
    x ^= x >> 15
    x = (x * 0x846CA68B) & M32
    x ^= x >> 16
    return x


def stream_key(seed, fmt, tile, op=0):
    return ct_mix(seed ^ ((((fmt * 16 + tile) * 2 + op) + 1) * 0x9E3779B9 & M32))


def kind(tile):
    return min(tile, 4)


def pattern(k, key, w):
    """The shared-memory test's data backgrounds (solid, checkerboard, alternating 128-byte rows, walking one, keyed),
    vectorized over the word index w."""
    w = np.asarray(w, dtype=np.uint64)
    if k == 0:
        return np.zeros(w.shape, dtype=np.uint64)
    if k == 1:
        return np.where(w & 1, 0xAAAAAAAA, 0x55555555).astype(np.uint64)
    if k == 2:
        return np.where((w >> 5) & 1, M32, 0).astype(np.uint64)
    if k == 3:
        return (np.uint64(1) << ((w + (w >> 5)) & 31)).astype(np.uint64)
    return ((w * PAT_MUL) & M32) ^ np.uint64(key)


def table(seed, fmt, tile):
    if fmt == DATA:
        return [kind(tile), stream_key(seed, 9, tile) if kind(tile) == 4 else 0, LINE_MUL if kind(tile) == 4 else 0, 37]
    if fmt == TEX:
        k = stream_key(seed, 7, tile)
        return [(k | 1) & (TEXELS - 1), (k >> 13) & (TEXELS - 1), (k >> 26) % 5, 0]
    return [tile % 4, stream_key(seed, 8, tile) & (WIN - 1), 0, 0]


# ---- L1_DATA ------------------------------------------------------------------------------------------------------
def writer(t, p):
    return (t - 32 * (p + 1)) % THREADS


def order(p, K):
    if p == 0:
        return list(range(K))
    if p == 1:
        return list(range(K - 1, -1, -1))
    return [b for r in range(4) for b in range(r, K, 4)]


def span_values(tab, K, c, inv=0):
    """The span of CTA c as written: every word with its background, line key and polarity."""
    w = np.arange(K * BLOCK, dtype=np.uint64)
    line = (c * K * BLOCK + w) // LINE
    key = ((line + 1) * tab[2]) & M32
    return pattern(tab[0], tab[1], w % BLOCK) ^ key ^ np.uint64(inv)


def data_reads(seed, tile, K, c=0):
    tab = table(seed, DATA, tile)
    span = span_values(tab, K, c)
    out = np.zeros((THREADS, 3, K, 4), dtype=np.uint64)
    for t in range(THREADS):
        for p in range(3):
            for s, b in enumerate(order(p, K)):
                out[t, p, s] = span[b * BLOCK + 4 * writer(t, p): b * BLOCK + 4 * writer(t, p) + 4]
    return out.reshape(THREADS, -1)


def _data_block_reads(tab, inv, fault):
    """What every thread reads from block 0 of CTA 0 (K = 1) in one repetition of polarity inv, [128, 12] raw, under a
    fault model."""
    span = span_values(tab, 1, 0, inv)
    stored = span.copy()
    name = fault[0] if fault else None
    if name == "alias":                      # line a answers for line b: b reads a's data
        _, a, b = fault
        stored[b * LINE:(b + 1) * LINE] = span[a * LINE:(a + 1) * LINE]
    elif name in ("stale", "sector"):        # the previous repetition's polarity is returned
        prev = span_values(tab, 1, 0, inv ^ M32)
        if name == "stale":
            stored = prev
        else:
            v = fault[1]
            stored[4 * v:4 * v + 4] = prev[4 * v:4 * v + 4]
    elif name in ("stuck0", "stuck1"):
        _, line, word, bit = fault
        i = line * LINE + word
        stored[i] = (stored[i] | (1 << bit)) if name == "stuck1" else (stored[i] & ~np.uint64(1 << bit) & M32)
    out = np.zeros((THREADS, 12), dtype=np.uint64)
    for t in range(THREADS):
        for p in range(3):
            out[t, 4 * p:4 * p + 4] = stored[4 * writer(t, p): 4 * writer(t, p) + 4]
    return out


def _data_fold(tab, reads):
    """The kernel's sum fold of one block: weight 2j + 1, the expected line key XORed out."""
    keys = np.zeros(12, dtype=np.uint64)
    out = []
    for t in range(THREADS):
        for p in range(3):
            keys[4 * p:4 * p + 4] = ((writer(t, p) // 8 + 1) * tab[2]) & M32
        h = 0
        for j in range(12):
            h += (2 * j + 1) * int(reads[t, j] ^ keys[j])
        out.append(h & M32)
    return out


# ---- L1_TEX -------------------------------------------------------------------------------------------------------
def texels(seed):
    """The image, [y][x][4]: the keyed background per texel word, rows y >= 64 complemented."""
    key = stream_key(seed, 10, 0)
    i = np.arange(TEXELS * 4, dtype=np.uint64)
    v = pattern(4, key, i).reshape(TEX_H, TEX_W, 4)
    v[TEX_H // 2:] ^= np.uint64(M32)
    return v


def tex_addr(mode, x, m, n):
    """The guide's address modes on the normalized coordinate u = (x + 1/2) / n + m, then point sampling floor(n u)."""
    u = (x + 0.5) / n + m
    if mode == WRAP:
        u = u - math.floor(u)
    elif mode == MIRROR:
        f = u - math.floor(u)
        u = f if math.floor(u) % 2 == 0 else 1 - f
    elif mode == CLAMP:
        u = 0.0 if u < 0 else (1 - 1 / n if u >= 1 else u)
    elif not 0 <= u < 1:
        return None
    return int(math.floor(u * n))


def _tex_addr_table(n):
    return {(mode, m): [tex_addr(mode, x, m, n) for x in range(n)] for mode in range(4) for m in range(-2, 3)}


_ADDR = {}


def results(seed, fmt, tile, fault=None):
    tab = table(seed, fmt, tile)
    if fmt == DATA:
        reads = _data_block_reads(tab, 0, fault)
        keys = np.array([[((writer(t, p) // 8 + 1) * tab[2]) & M32 for p in range(3) for _ in range(4)]
                         for t in range(THREADS)], dtype=np.uint64)
        return (reads ^ keys).astype(np.uint64)
    if fmt == TEX:
        return _tex_results(seed, tab, fault)
    return _const_results(seed, tab, fault)


def _tex_results(seed, tab, fault):
    img = texels(seed)
    A, B, D = tab[0], tab[1], tab[2]
    if not _ADDR:
        _ADDR[TEX_W] = _tex_addr_table(TEX_W)
        _ADDR[TEX_H] = _tex_addr_table(TEX_H)
    out = np.zeros((THREADS, STEPS, 8, 4), dtype=np.uint64)
    zero = np.zeros(4, dtype=np.uint64)
    for t in range(THREADS):
        for j in range(STEPS):
            i = (A * (THREADS * j + t) + B) & (TEXELS - 1)
            x, y = i % TEX_W, i // TEX_W
            mx, my = (t + j + D) % 5 - 2, (t // 5 + 2 * j + 3 * D) % 5 - 2
            # x and y swapped: tld reads column y (clamped, as object 0 clamps) of row x
            out[t, j, 0] = img[x, min(y, TEX_W - 1)] if fault == "swap_xy" else img[y, x]
            out[t, j, 1] = img[(y + 1) % TEX_H, x] if fault == "next_row" else img[y, x]
            for mode in range(4):
                md = mode
                if fault == "wrap_as_clamp" and mode == WRAP:
                    md = CLAMP
                if fault == "border_as_edge" and mode == BORDER:
                    md = CLAMP
                ix, iy = _ADDR[TEX_W][(md, mx)][x], _ADDR[TEX_H][(md, my)][y]
                if fault == "mirror_off_by_one" and mode == MIRROR:
                    ix = (TEX_W - x) % TEX_W if mx % 2 else x
                    iy = (TEX_H - y) % TEX_H if my % 2 else y
                out[t, j, 2 + mode] = zero if ix is None or iy is None else img[iy, ix]
            c = j % 4
            x1, y1 = min(x + 1, TEX_W - 1), min(y + 1, TEX_H - 1)
            g = [img[y1, x, c], img[y1, x1, c], img[y, x1, c], img[y, x, c]]   # (i0,j1) (i1,j1) (i1,j0) (i0,j0)
            if fault == "tld4_rotated":
                g = g[1:] + g[:1]
            out[t, j, 6] = g
            out[t, j, 7] = img[y, x]
    return out.reshape(THREADS, -1)


# ---- L1_CONST -----------------------------------------------------------------------------------------------------
def bank(seed):
    key = stream_key(seed, 11, 0)
    k = np.arange(BANK, dtype=np.uint64)
    w = k // WIN
    v = pattern(4, key, (w & 1) * WIN + k % WIN)
    v[w >= 2] ^= np.uint64(M32)
    return v


def _const_results(seed, tab, fault):
    C = bank(seed)
    base, rot = tab[0] * WIN, tab[1]
    out = []
    for t in range(THREADS):
        w, lane = t // 32, t % 32
        uni = [(k + 512 * w + rot) % WIN for k in range(WIN)]
        div = [(64 * (0 if fault == "divergent_as_lane0" else lane) + k + 512 * w + rot) % WIN for k in range(64)]
        v2 = [(2 * (32 * lane + k) + 512 * w + 2 * rot) % WIN + e for k in range(32) for e in range(2)]
        v4 = [(4 * (16 * lane + k) + 512 * w + 4 * rot) % WIN + e for k in range(16) for e in range(4)]
        idx = np.array([base + i for i in uni + div + v2 + v4], dtype=np.int64)
        if fault == "wrong_window":
            idx[0] = (idx[0] + WIN) % BANK
        r = C[idx]
        if fault == "stuck_bit":
            r = r | np.uint64(1 << 13)
        out.append(r)
    return np.array(out, dtype=np.uint64)


# ---- folds and checks ---------------------------------------------------------------------------------------------
def it_fold_rows(words):
    """it_fold of every row of words [n, W]: four multiply-and-rotate chains, word i to chain i % 4."""
    words = np.asarray(words, dtype=np.uint64)
    h = [np.full(words.shape[0], v, dtype=np.uint64) for v in FOLD_INIT]
    for i in range(words.shape[1]):
        x = ((h[i & 3] ^ words[:, i]) * np.uint64(FOLD_MUL)) & np.uint64(M32)
        h[i & 3] = ((x << np.uint64(FOLD_ROT)) | (x >> np.uint64(32 - FOLD_ROT))) & np.uint64(M32)

    def rotl(v, n):
        return ((v << np.uint64(n)) | (v >> np.uint64(32 - n))) & np.uint64(M32)
    return [int(v) for v in h[0] ^ rotl(h[1], 8) ^ rotl(h[2], 16) ^ rotl(h[3], 24)]


def sum_fold(words):
    return sum((2 * j + 1) * int(w) for j, w in enumerate(words)) & M32


def checks(seed, fmt, tile, fault=None):
    """Per thread: the host's check (L1_TEX / L1_CONST), or (even, odd) block folds of L1_DATA at K = 1."""
    if fmt == DATA:
        tab = table(seed, fmt, tile)
        return list(zip(_data_fold(tab, _data_block_reads(tab, 0, fault)),
                        _data_fold(tab, _data_block_reads(tab, M32, fault))))
    return it_fold_rows(results(seed, fmt, tile, fault))


FAULTS = {
    DATA: [("stuck%d" % v, line, 5, bit) for v in (0, 1) for line in (0, 7, 15) for bit in range(32)]
    + [("alias", 0, 2), ("stale",), ("sector", 9)],
    TEX: ["wrap_as_clamp", "mirror_off_by_one", "border_as_edge", "swap_xy", "tld4_rotated", "next_row"],
    CONST: ["divergent_as_lane0", "wrong_window", "stuck_bit"],
}
# aliasing lines 0 and 2 of a block is invisible where both lines hold the same background and no line key: the solid,
# checkerboard and alternating-row tiles
VISIBLE = {fmt: {f: set(range(TILES)) for f in FAULTS[fmt]} for fmt in FAULTS}
VISIBLE[DATA][("alias", 0, 2)] = {3, 4, 5, 6, 7}
