"""Numpy restatement of the register-file self-test's host arithmetic (csrc/rf_test_math.hpp) and a model of its three
marches (csrc/rf_selftest.cuh) over every thread's held registers, with optional faults.

march() runs one comparison -- one march of one tile -- element by element on a RegFile of [THREADS, HELD] 32-bit
registers.  An element is its reads (every held register, in the element's order, compared and folded), then its
writes (an in-place ALU transition of the value read, or a quad / pair load of the next value); a fault model sees
the writes of an element after all of its reads.  It returns the final registers, every thread's fold and the OR of
its direct-compare differences (the kernel's DUMP), and optionally every value each thread read.
"""
import numpy as np

TILES, THREADS, REPS = 8, 128, 16
ALU, LOAD, HOLD = 0, 1, 2
FORMATS = (ALU, LOAD, HOLD)
NAMES = {ALU: "alu", LOAD: "load", HOLD: "hold"}
HELD = 204
ELEMENTS = {ALU: 6, LOAD: 5, HOLD: 3}
READS = {ALU: 5, LOAD: 4, HOLD: 2}
WRITES = {ALU: 5, LOAD: 4, HOLD: 2}
TABLE_WORDS = 5
HOOK_REG, HOOK_ELEMENT, HOOK_THREAD = HELD // 2, 0, 0
PARAM_WORDS = 12
SMEM_BYTES = 4 * (PARAM_WORDS + 2 * THREADS + HELD * THREADS)
DUMP_WORDS = HELD * THREADS + 2 * THREADS
HOLD_NS = 100000
PATTERN_MUL = 2654435761
M32 = 0xFFFFFFFF
T = np.arange(THREADS, dtype=np.uint64)[:, None]
J = np.arange(HELD, dtype=np.uint64)[None, :]


def bytes_per_tile(fmt: int) -> int:
    return 4 * HELD * THREADS * (READS[fmt] + WRITES[fmt])


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
    return stream_key(seed, 6 + fmt, tile, 0) if kind(tile) == 4 else 0


def pattern(kd: int, ky: int, t=T, j=J) -> np.ndarray:
    """P(t, j) as uint32, broadcast over thread and register indices."""
    t, j = np.broadcast_arrays(np.asarray(t, np.uint64), np.asarray(j, np.uint64))
    if kd == 0:
        return np.zeros(t.shape, np.uint32)
    if kd == 1:
        return np.where(j & np.uint64(1), np.uint64(0xAAAAAAAA), np.uint64(0x55555555)).astype(np.uint32)
    if kd == 2:
        return np.where(j & np.uint64(1), np.uint64(M32), np.uint64(0)).astype(np.uint32)
    if kd == 3:
        return (np.uint64(1) << ((t + j) & np.uint64(31))).astype(np.uint32)
    w = t * np.uint64(HELD) + j
    return (((w * np.uint64(PATTERN_MUL)) & np.uint64(M32)) ^ np.uint64(ky)).astype(np.uint32)


def fold(values) -> int:
    v = np.asarray(values, dtype=np.uint64)
    return int(((v * (2 * np.arange(v.size, dtype=np.uint64) + 1)).sum()) & np.uint64(M32))


def tables(seed: int, fmt: int) -> np.ndarray:
    return np.array([[kind(t), key(seed, fmt, t), HOOK_REG, HOOK_ELEMENT, HOOK_THREAD] for t in range(TILES)],
                    dtype=np.uint32)


# ---- the register file and its faults -----------------------------------------------------------------------------
class RegFile:
    """Every thread's held registers, [THREADS, HELD] uint32.  write() takes the whole file's new values and the port
    that writes them ("alu", "load4", "load2"); a subclass overrides _store / _load for a fault."""

    def __init__(self, init=None):
        self.r = np.zeros((THREADS, HELD), np.uint32) if init is None else np.array(init, np.uint32)

    def _store(self, new, port):
        self.r = new.astype(np.uint32)

    def _load(self):
        return self.r.copy()

    def write(self, new, port):
        self._store(np.asarray(new, np.uint32), port)

    def read(self):
        return self._load()

    def hold(self, n):
        """The n-th hold interval of RF_HOLD passes."""

    def flip(self, t, j, mask):
        self.r[t, j] ^= np.uint32(mask)


class Stuck(RegFile):
    """Bits in `mask` ([THREADS, HELD] uint32) read and keep `value`'s bits there, whatever is written."""

    def __init__(self, mask, value, init=None):
        super().__init__(init)
        self.mask, self.value = mask.astype(np.uint32), value.astype(np.uint32)
        self.r = (self.r & ~self.mask) | (self.value & self.mask)

    def _store(self, new, port):
        self.r = (new & ~self.mask) | (self.value & self.mask)


class Transition(RegFile):
    """Bits in `up` cannot rise (a 0 stays 0 when 1 is written); bits in `down` cannot fall."""

    def __init__(self, up, down, init=None):
        super().__init__(init)
        self.up, self.down = up.astype(np.uint32), down.astype(np.uint32)

    def _store(self, new, port):
        old = self.r
        blocked = (self.up & ~old & new) | (self.down & old & ~new)
        self.r = (new ^ blocked).astype(np.uint32)


class Misroute(RegFile):
    """A write to register j of thread t lands in register j2 instead (j keeps its value)."""

    def __init__(self, t, j, j2, init=None):
        super().__init__(init)
        self.t, self.j, self.j2 = t, j, j2

    def _store(self, new, port):
        new = new.copy()
        new[self.t, self.j2] = new[self.t, self.j]
        new[self.t, self.j] = self.r[self.t, self.j]
        self.r = new


class LaneDrop(RegFile):
    """A load of `width` registers (4: a quad, 2: a pair) into register j of thread t does not write it."""

    def __init__(self, t, j, width, init=None):
        super().__init__(init)
        self.t, self.j, self.width = t, j, width

    def _store(self, new, port):
        new = new.copy()
        if port == "load%d" % self.width:
            new[self.t, self.j] = self.r[self.t, self.j]
        self.r = new


class HoldFlip(RegFile):
    """Register j of thread t flips the bits of `mask` during hold interval n."""

    def __init__(self, t, j, mask, n, init=None):
        super().__init__(init)
        self.t, self.j, self.mask, self.n = t, j, mask, n

    def hold(self, n):
        if n == self.n:
            self.flip(self.t, self.j, self.mask)


def steady(fmt, kd, ky):
    """The registers a clean repetition leaves for the next one of the same tile: P (RF_ALU) or ~P."""
    p = pattern(kd, ky)
    return p if fmt == ALU else p ^ np.uint32(M32)


# ---- the marches ----------------------------------------------------------------------------------------------------
def march(fmt, kd, ky, rf=None, hook=None, keep_reads=False):
    """One comparison of format fmt on tile (kd, ky).  rf defaults to a clean file holding what the previous
    repetition left (steady()).  hook = (element, thread, register, mask): after that element, XOR mask into that
    register.  Returns a dict: regs ([THREADS, HELD] after the march), fold and err ([THREADS]: the fold of the reads
    and the OR of their differences from the pattern), reads (keep_reads: [THREADS, n] in read order)."""
    rf = rf if rf is not None else RegFile(steady(fmt, kd, ky))
    p = pattern(kd, ky)
    h = np.zeros(THREADS, np.uint64)
    err = np.zeros(THREADS, np.uint32)
    log = []
    n_read = 0

    def read(inv, down):
        nonlocal h, err, n_read
        v = rf.read()
        order = slice(None, None, -1) if down else slice(None)
        got, want = v[:, order], (p ^ np.uint32(inv))[:, order]
        w = 2 * (n_read + np.arange(HELD, dtype=np.uint64)) + 1
        h = (h + (got.astype(np.uint64) * w).sum(axis=1)) & np.uint64(M32)
        err |= np.bitwise_or.reduce(got ^ want, axis=1)
        n_read += HELD
        if keep_reads:
            log.append(got)
        return v

    def alu(v):
        rf.write(v ^ np.uint32(M32), "alu")

    def elements():
        """Yields once per element, after it ran (the hook and the holds go there)."""
        if fmt == ALU:
            rf.write(p, "load4")
            yield
            for inv, down in ((0, False), (M32, False), (0, True), (M32, True)):
                alu(read(inv, down))
                yield
            read(0, False)
            yield
        elif fmt == LOAD:
            rf.write(p, "load4")
            yield
            for inv, port in ((0, "load4"), (M32, "load2"), (0, "load2")):
                read(inv, False)
                rf.write(p ^ np.uint32(inv ^ M32), port)
                yield
            read(M32, False)
            yield
        else:
            rf.write(p, "load4")
            yield
            alu(read(0, False))
            yield
            read(M32, False)
            yield

    holds = 0
    for e, _ in enumerate(elements()):
        if hook is not None and hook[0] == e:
            rf.flip(hook[1], hook[2], hook[3])
        if fmt == HOLD and e < ELEMENTS[HOLD] - 1:
            rf.hold(holds)
            holds += 1
    out = {"regs": rf.read(), "fold": h.astype(np.uint32), "err": err}
    if keep_reads:
        out["reads"] = np.concatenate(log, axis=1)
    return out


def checks(seed: int, fmt: int) -> np.ndarray:
    """[TILES][THREADS] check values: every thread's fold of a clean march."""
    return np.stack([march(fmt, kind(t), key(seed, fmt, t))["fold"] for t in range(TILES)])
