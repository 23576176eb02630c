"""Numpy restatement of the shared-memory self-test's host arithmetic (csrc/smem_test_math.hpp) and a model of its
three marches (csrc/smem_selftest.cuh) over a byte-addressed array, with optional faults.

march() runs one comparison -- one march of one tile -- step by step: every element walks k in its direction, and at
each k all 128 threads make their access at once (each cell is touched once per element, so the order between threads
only matters to a fault that couples two addresses).  It returns the final image, every thread's fold and
direct-compare error count, the bytes each element touched, and an error-bit map that attributes every wrong read to
the bytes it came from.  SH_DSMEM models a pair of arrays; the two ranks run each element one after the other, in the
order `order` gives.
"""
import numpy as np

TILES, THREADS, REPS = 8, 128, 16
WORD, BYTE, DSMEM = 0, 1, 2
FORMATS = (WORD, BYTE, DSMEM)
NAMES = {WORD: "word", BYTE: "byte", DSMEM: "dsmem"}
BYTES = 232448
WORDS = BYTES // 4                 # 58,112
WPT = WORDS // THREADS             # 454 words per thread
VECS, VPT, VTAIL = BYTES // 16, BYTES // 16 // THREADS, BYTES // 16 % THREADS   # 14,528, 113, 64
PPT = BYTES // 8 // THREADS        # 227 pairs per thread
ELEMENTS = {WORD: 6, BYTE: 4, DSMEM: 4}
HOOK_WORD, HOOK_ELEMENT = 4660, 0
TABLE_WORDS = 4
DUMP_WORDS = WORDS + 2 * THREADS
PATTERN_MUL = 2654435761
BYTES_PER_TILE = {WORD: 10 * BYTES, BYTE: 6 * BYTES, DSMEM: 6 * BYTES}
M32 = 0xFFFFFFFF
T = np.arange(THREADS, dtype=np.int64)


def mix(x: int) -> int:
    x &= M32
    x ^= x >> 16
    x = (x * 0x7FEB352D) & M32
    x ^= x >> 15
    x = (x * 0x846CA68B) & M32
    x ^= x >> 16
    return x


def stream_key(seed: int, fmt: int, tile: int, op: int) -> int:
    return mix(seed ^ ((((fmt * 16 + tile) * 2 + op) + 1) * 0x9E3779B9 & M32))


def kind(tile: int) -> int:
    return tile if tile < 4 else 4


def key(seed: int, fmt: int, tile: int) -> int:
    return stream_key(seed, 3 + fmt, tile, 0) if kind(tile) == 4 else 0


def pattern(kd: int, ky: int, w) -> np.ndarray:
    """P(w) as uint32 for an array of word indices."""
    w = np.asarray(w, dtype=np.uint64)
    if kd == 0:
        return np.zeros(w.shape, np.uint32)
    if kd == 1:
        return (np.uint64(0x55555555) ^ np.where(w & np.uint64(1), np.uint64(M32), np.uint64(0))).astype(np.uint32)
    if kd == 2:
        return np.where((w >> np.uint64(5)) & np.uint64(1), np.uint64(M32), np.uint64(0)).astype(np.uint32)
    if kd == 3:
        return (np.uint64(1) << ((w + (w >> np.uint64(5))) & np.uint64(31))).astype(np.uint32)
    return (((w * np.uint64(PATTERN_MUL)) & np.uint64(M32)) ^ np.uint64(ky)).astype(np.uint32)


def rank_key(r: int) -> int:
    return ((r + 1) * 0x9E3779B9) & M32


def fold(values) -> int:
    v = np.asarray(values, dtype=np.uint64)
    return int(((v * (2 * np.arange(v.size, dtype=np.uint64) + 1)).sum()) & np.uint64(M32))


def tables(seed: int, fmt: int) -> np.ndarray:
    return np.array([[kind(t), key(seed, fmt, t), HOOK_WORD, HOOK_ELEMENT] for t in range(TILES)], dtype=np.uint32)


# ---- the array and its faults -------------------------------------------------------------------------------------
class Mem:
    """A byte-addressed array.  write / read take [n] byte addresses of n accesses of `width` bytes; `remote` marks a
    DSMEM store from the peer CTA.  A subclass overrides _store / _load for a fault."""

    def __init__(self, init=None):
        self.b = np.zeros(BYTES, np.uint8) if init is None else np.array(init, dtype=np.uint8).copy()

    def _store(self, addr, data, width, remote):
        self.b[addr[:, None] + np.arange(width)] = data

    def _load(self, addr, width):
        return self.b[addr[:, None] + np.arange(width)]

    def write(self, addr, data, width, remote=False):
        self._store(np.asarray(addr, np.int64), data, width, remote)

    def read(self, addr, width):
        return self._load(np.asarray(addr, np.int64), width)

    def words(self):
        return self.b.view("<u4").copy()


class Stuck(Mem):
    """Bytes in `mask` (uint8 [BYTES]) read and keep `value`'s bits there, whatever is written."""

    def __init__(self, mask, value, init=None):
        super().__init__(init)
        self.mask, self.value = mask.astype(np.uint8), value.astype(np.uint8)
        self._fix(np.arange(BYTES))

    def _fix(self, idx):
        self.b[idx] = (self.b[idx] & ~self.mask[idx]) | (self.value[idx] & self.mask[idx])

    def _store(self, addr, data, width, remote):
        super()._store(addr, data, width, remote)
        self._fix((addr[:, None] + np.arange(width)).ravel())


class Transition(Mem):
    """Bits in `up` cannot rise (a 0 stays 0 when 1 is written); bits in `down` cannot fall (uint8 [BYTES] masks)."""

    def __init__(self, up, down, init=None):
        super().__init__(init)
        self.up, self.down = up.astype(np.uint8), down.astype(np.uint8)

    def _store(self, addr, data, width, remote):
        idx = addr[:, None] + np.arange(width)
        old, new = self.b[idx], data.astype(np.uint8)
        blocked = (self.up[idx] & ~old & new) | (self.down[idx] & old & ~new)
        self.b[idx] = new ^ blocked


class Alias(Mem):
    """Word a of each pair (a, b) reaches word b's cell."""

    def __init__(self, pairs, init=None):
        super().__init__(init)
        self.remap = np.arange(BYTES, dtype=np.int64)
        for a, b in pairs:
            self.remap[4 * a:4 * a + 4] = np.arange(4 * b, 4 * b + 4)

    def _store(self, addr, data, width, remote):
        self.b[self.remap[addr[:, None] + np.arange(width)]] = data

    def _load(self, addr, width):
        return self.b[self.remap[addr[:, None] + np.arange(width)]]


class ByteSpill(Mem):
    """A st.u8 to byte f also writes its value to byte f + d."""

    def __init__(self, f, d, init=None):
        super().__init__(init)
        self.f, self.d = f, d

    def _store(self, addr, data, width, remote):
        super()._store(addr, data, width, remote)
        if width == 1:
            hit = addr == self.f
            if hit.any():
                self.b[self.f + self.d] = data[hit][0, 0]


class LaneDrop(Mem):
    """A store of `width` bytes that covers byte f does not write the lane holding f (a byte of st.u16, a word of
    st.v4)."""

    def __init__(self, f, width, init=None):
        super().__init__(init)
        self.f, self.width = f, width

    def _store(self, addr, data, width, remote):
        if width != self.width:
            return super()._store(addr, data, width, remote)
        lane = 1 if width == 2 else 4
        idx = addr[:, None] + np.arange(width)
        keep = ~((idx // lane) == (self.f // lane))
        self.b[idx[keep]] = data[keep]


class RemoteFault(Mem):
    """DSMEM: a remote store into word w of this array is lost (lost=True), or lands in the writer's own array at the
    same address (`own`, the writer's Mem)."""

    def __init__(self, w, lost, init=None):
        super().__init__(init)
        self.w, self.lost, self.own = w, lost, None

    def _store(self, addr, data, width, remote):
        hit = (addr // 4 == self.w) if remote else np.zeros(addr.shape, bool)
        super()._store(addr[~hit], data[~hit], width, remote)
        if hit.any() and not self.lost:
            Mem._store(self.own, addr[hit], data[hit], width, False)


# ---- the marches --------------------------------------------------------------------------------------------------
def _le(words: np.ndarray, width: int) -> np.ndarray:
    """[n] uint32 -> [n, width] little-endian bytes of the low `width` bytes (width <= 4)."""
    return np.stack([(words >> np.uint32(8 * i)) & np.uint32(0xFF) for i in range(width)], axis=1).astype(np.uint8)


def _words(b: np.ndarray) -> np.ndarray:
    """[n, 4 m] bytes -> [n, m] uint32."""
    return np.ascontiguousarray(b).view("<u4").reshape(b.shape[0], -1)


class _Thread:
    """Every thread's read log: fold, error count, optional list of values; and the error-bit map of one array."""

    def __init__(self, keep):
        self.h = np.zeros(THREADS, np.uint64)
        self.j = np.zeros(THREADS, np.uint64)
        self.err = np.zeros(THREADS, np.int64)
        self.log = [[] for _ in range(THREADS)] if keep else None

    def take(self, th, got, want, fk=0):
        """th [n] threads; got / want [n] values (uint32) read / expected; fk XORed out before the fold."""
        v = (got.astype(np.uint64) ^ np.uint64(fk)) & np.uint64(M32)
        self.h[th] = (self.h[th] + (2 * self.j[th] + 1) * v) & np.uint64(M32)
        self.j[th] += 1
        self.err[th] += got != want
        if self.log is not None:
            for t, x in zip(th.tolist(), v.tolist()):
                self.log[t].append(x)


def march(fmt, kd, ky, mem=None, peer=None, hook=None, order=(0, 1), keep_reads=False):
    """One comparison of format fmt on tile (kd, ky).  mem (and for DSMEM peer: rank 1's array) default to clean
    zeroed arrays.  hook = (rank, element, word, mask): after that element, XOR mask into that word of that rank's
    array.  Returns a dict: image (uint32 words; DSMEM: a list per rank), fold / err per thread (DSMEM: per rank),
    errmap (uint8 [BYTES] per rank: the bits some read got wrong), touched (per element, the bytes it touched per
    rank), reads (keep_reads: per rank, per thread, the values folded)."""
    mems = [mem or Mem()] + ([peer or Mem()] if fmt == DSMEM else [])
    for m in mems:
        if isinstance(m, RemoteFault):
            m.own = mems[1 - mems.index(m)]
    ranks = len(mems)
    logs = [_Thread(keep_reads) for _ in range(ranks)]
    errmap = [np.zeros(BYTES, np.uint8) for _ in range(ranks)]
    touched = []
    P = lambda w: pattern(kd, ky, w)  # noqa: E731

    def note(r, addr, got, want):
        bad = np.bitwise_xor(got, want).astype(np.uint8)
        np.bitwise_or.at(errmap[r], addr, bad)

    def elem_word(r, target, up, read_inv, write_inv, rk, tc):
        """A word element of rank r on array `target`: reads expect P ^ read_inv ^ rk (None: no read), writes store
        P ^ write_inv ^ rk (None: no write); the fold removes rk."""
        m = mems[target]
        for i in range(WPT):
            k = i if up else WPT - 1 - i
            w = T + THREADS * k
            addr = 4 * w
            tc[target][(addr[:, None] + np.arange(4)).ravel()] += 1
            p = P(w)
            if read_inv is not None:
                want = p ^ np.uint32(read_inv ^ rk)
                got = _words(m.read(addr, 4))[:, 0]
                note(target, (addr[:, None] + np.arange(4)).ravel(), _le(got, 4).ravel(), _le(want, 4).ravel())
                logs[r].take(T, got, want, rk)
            if write_inv is not None:
                m.write(addr, _le(p ^ np.uint32(write_inv ^ rk), 4), 4, remote=target != r)

    nv = VPT + (T < VTAIL)

    def elements():
        """Yields once per element, after it ran (the hook and the touch record go there)."""
        if fmt == WORD:
            for up, ri, wi in ((True, None, 0), (True, 0, M32), (True, M32, 0), (False, 0, M32), (False, M32, 0),
                               (True, 0, None)):
                tc = [np.zeros(BYTES, np.int64)]
                elem_word(0, 0, up, ri, wi, 0, tc)
                yield tc
        elif fmt == BYTE:
            m = mems[0]
            tc = [np.zeros(BYTES, np.int64)]
            for k in range(WPT):
                w = T + THREADS * k
                p = P(w)
                for b in (3, 0, 2, 1):
                    tc[0][4 * w + b] += 1
                    m.write(4 * w + b, _le(p >> np.uint32(8 * b), 1), 1)
            yield tc
            tc = [np.zeros(BYTES, np.int64)]
            for k in range(VPT + 1):
                th = T[k < nv]
                v = th + THREADS * k
                addr = 16 * v
                tc[0][(addr[:, None] + np.arange(16)).ravel()] += 1
                got = _words(m.read(addr, 16))
                want = P((4 * v)[:, None] + np.arange(4))
                note(0, (addr[:, None] + np.arange(16)).ravel(), _le(got.ravel(), 4).ravel(), _le(want.ravel(), 4).ravel())
                for i in range(4):
                    logs[0].take(th, got[:, i], want[:, i])
                for i in range(4):
                    inv = ~want[:, i]
                    m.write(addr + 4 * i, _le(inv, 2), 2)
                    m.write(addr + 4 * i + 2, _le(inv >> np.uint32(16), 2), 2)
            yield tc
            tc = [np.zeros(BYTES, np.int64)]
            for k in range(VPT, -1, -1):
                th = T[k < nv]
                v = th + THREADS * k
                addr = 16 * v
                tc[0][(addr[:, None] + np.arange(16)).ravel()] += 1
                p = P((4 * v)[:, None] + np.arange(4))
                got = m.read(addr, 16)
                want = _le((~p).ravel(), 4).reshape(len(th), 16)
                note(0, (addr[:, None] + np.arange(16)).ravel(), got.ravel(), want.ravel())
                for i in range(16):
                    logs[0].take(th, got[:, i].astype(np.uint32), want[:, i].astype(np.uint32))
                m.write(addr, _le(p.ravel(), 4).reshape(len(th), 16), 16)
            yield tc
            tc = [np.zeros(BYTES, np.int64)]
            for k in range(PPT - 1, -1, -1):
                u = T + THREADS * k
                addr = 8 * u
                tc[0][(addr[:, None] + np.arange(8)).ravel()] += 1
                got = _words(m.read(addr, 8))
                want = P((2 * u)[:, None] + np.arange(2))
                note(0, (addr[:, None] + np.arange(8)).ravel(), _le(got.ravel(), 4).ravel(), _le(want.ravel(), 4).ravel())
                logs[0].take(T, got[:, 0], want[:, 0])
                logs[0].take(T, got[:, 1], want[:, 1])
            yield tc
        else:
            rk = [rank_key(0), rank_key(1)]
            for remote, ri, wi in ((True, None, 0), (False, 0, M32), (True, M32, 0), (False, 0, None)):
                tc = [np.zeros(BYTES, np.int64), np.zeros(BYTES, np.int64)]
                for r in order:
                    target = 1 - r if remote else r
                    elem_word(r, target, True, ri, wi, rk[target], tc)
                yield tc

    for e, tc in enumerate(elements()):
        touched.append(tc)
        if hook is not None and hook[1] == e:
            r, _, w, mask = hook
            cur = _words(mems[r].read(np.array([4 * w]), 4))[:, 0] ^ np.uint32(mask)
            mems[r].write(np.array([4 * w]), _le(cur, 4), 4)
    out = {"image": [m.words() for m in mems], "fold": [lg.h.astype(np.uint32) for lg in logs],
           "err": [lg.err for lg in logs], "errmap": errmap, "touched": touched}
    if keep_reads:
        out["reads"] = [lg.log for lg in logs]
    if fmt != DSMEM:
        for k in ("image", "fold", "err", "errmap"):
            out[k] = out[k][0]
    return out


def checks(seed: int, fmt: int) -> np.ndarray:
    """[TILES][THREADS] check values: every thread's fold of a clean march."""
    out = np.zeros((TILES, THREADS), np.uint32)
    for t in range(TILES):
        r = march(fmt, kind(t), key(seed, fmt, t))
        out[t] = r["fold"][0] if fmt == DSMEM else r["fold"]
    return out
