"""Oracle for the on-demand memory test (numpy; test infrastructure only).

The specification of the arithmetic the CUDA march (k8s-device-plugin_b200/csrc/hbm_memtest.cuh) and its host side
(csrc/memtest_math.hpp) must reproduce bit for bit.  It builds on the probe oracle (oracle/probe.py):

    segment seed    : seed_g = seed ^ uint32(g * 0x9E3779B9)
    word i          : (uint32(i) * 2654435761) ^ seed_g      i = global word index over the concatenated segments
    march           : E0 w(P)   E1 r(P) w(~P)   E2 r(~P) w(P)   E3 r(P)       ~P = the pattern under ~seed_g
    element k       : checksum   = sum of the words read             mod 2^64   (0 for E0, which reads nothing)
                      mismatches = #{ i : word read != expected }
                      first_bad  = min such i, else 2^64-1
    faults          : (word, mask) XORs applied right after E0
    plan            : min(max, free - reserve) rounded down to 2 MiB, in 1 GiB segments (the last may be smaller),
                      at most 256 of them; reserve 0 = total // 10, max 0 = no cap
"""
import numpy as np

from oracle import probe as oprobe

CHUNK_BYTES = 1 << 30
ALIGN_BYTES = 2 << 20
MAX_SEGMENTS = 256
INV = 0xFFFFFFFF
NO_BAD = oprobe.NO_BAD
# (reads, writes, inv, delta) per element: the expected pattern is keyed with seed_g ^ inv, the word written is
# (word read) ^ delta
MARCH = [(False, True, 0, 0), (True, True, 0, INV), (True, True, INV, INV), (True, False, 0, 0)]


def default_reserve(total_bytes: int) -> int:
    return total_bytes // 10


def segment_seed(seed: int, g: int) -> int:
    return (seed ^ ((g * 0x9E3779B9) & 0xFFFFFFFF)) & 0xFFFFFFFF


def plan(free_bytes: int, total_bytes: int, reserve_bytes: int = 0, max_bytes: int = 0):
    """Segment sizes in bytes (csrc/memtest_math.hpp memtest_plan)."""
    reserve = reserve_bytes or default_reserve(total_bytes)
    budget = max(0, free_bytes - reserve)
    if max_bytes:
        budget = min(budget, max_bytes)
    budget = min(budget, CHUNK_BYTES * MAX_SEGMENTS)
    budget -= budget % ALIGN_BYTES
    out = []
    while budget:
        s = min(budget, CHUNK_BYTES)
        out.append(s)
        budget -= s
    return out


def range_checksum(base: int, n: int, seed: int, chunk: int = 1 << 24) -> int:
    """Sum of word(i, seed) over base <= i < base + n, mod 2^64, by summing the pattern with numpy."""
    total = 0
    for start in range(0, n, chunk):
        m = min(chunk, n - start)
        total = (total + oprobe.checksum(oprobe.pattern(m, seed, base + start))) & NO_BAD
    return total


def expected_checksum(segments_words, seed: int, inv: int = 0) -> int:
    """What a clean reading element sums to over the segments (word counts, in order)."""
    total, base = 0, 0
    for g, n in enumerate(segments_words):
        total = (total + range_checksum(base, n, segment_seed(seed, g) ^ inv)) & NO_BAD
        base += n
    return total


def _seeds(segments_words, seed):
    return np.concatenate([np.full(n, segment_seed(seed, g), dtype=np.uint32) for g, n in enumerate(segments_words)])


def march(segments_words, seed: int, faults=()):
    """The four elements over segments of the given word counts -> one (checksum, mismatches, first_bad, buffer
    after the element) per element; the buffer is the concatenation of the segments."""
    n = int(sum(segments_words))
    base = oprobe.pattern(n, 0)                    # uint32(i) * K
    seeds = _seeds(segments_words, seed)
    buf = None
    out = []
    for k, (reads, writes, inv, delta) in enumerate(MARCH):
        exp = base ^ (seeds ^ np.uint32(inv))
        if not reads:
            buf = exp.copy()
            out.append((0, 0, NO_BAD, buf.copy()))
            for w, mask in faults:
                buf[w] ^= np.uint32(mask)
            continue
        bad = np.nonzero(buf != exp)[0]
        cs = oprobe.checksum(buf)
        if writes:
            buf = buf ^ np.uint32(delta)
        out.append((cs, int(bad.size), int(bad[0]) if bad.size else NO_BAD, buf.copy()))
    return out


def memtest_healthy(launch_ok: bool, mismatches, checksums, expected, ecc_uncorrected: int, remap_failed: bool,
                    remap_pending: bool) -> bool:
    """The verdict (csrc/memtest_math.hpp memtest_healthy): the launches succeeded, every reading element (1-3) has no
    mismatch and the closed-form checksum, no uncorrected ECC error appeared and no row remap failed or is pending.
    Corrected ECC errors do not fail a device."""
    if not launch_ok or ecc_uncorrected or remap_failed or remap_pending:
        return False
    return all(mismatches[k] == 0 and checksums[k] == expected[k] for k in (1, 2, 3))
