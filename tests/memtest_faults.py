"""Faulty-memory oracle for the memory-test march (numpy; test infrastructure only).

tests/memtest_oracle.py models a healthy memory with XORs applied right after E0.  This module models the march of
k8s-device-plugin_b200/csrc/hbm_memtest.cuh as it is written over memory with faulty cells:

    E0  writes P
    E1  reads, compares with P,  writes (word read) ^ 0xFFFFFFFF
    E2  reads, compares with ~P, writes (word read) ^ 0xFFFFFFFF
    E3  reads, compares with P

E1 and E2 write back the word they READ, re-keyed, not the word they expected, so a wrong read carries forward into
every later element.  A fault is (word, model, mask); after each writing element the faulty word holds
cell_after_write(model, mask, elem, before, written).  The models act on the bits of `mask`:

    xor@k     one flip after element k (k = 0, 1, 2); xor@0 is memtest_oracle.march's fault
    stuck0/1  the bit always holds 0 / 1
    tf_up     a write that would move the bit 0 -> 1 leaves it at 0; 1 -> 0 and writes of the same value work
    tf_down   a write that would move the bit 1 -> 0 leaves it at 1; 0 -> 1 and writes of the same value work

The buffer reported after an element is what the element wrote, before the faulty cells act on it, so the GPU test
compares the kernel's own stores with the oracle and then applies the same function to the device words."""
from typing import NamedTuple

import numpy as np

import memtest_oracle as mt
from oracle import probe as oprobe

MODELS = ("xor@0", "xor@1", "xor@2", "stuck0", "stuck1", "tf_up", "tf_down")
CELL_MODELS = ("stuck0", "stuck1", "tf_up", "tf_down")


class Fault(NamedTuple):
    word: int           # global word index over the concatenated segments
    model: str          # one of MODELS
    mask: int           # the faulty bits (nonzero)


def cell_after_write(model, mask, elem, before, written):
    """What faulty cells hold after march element `elem` wrote `written` over `before` (uint32 scalars or arrays)."""
    mask, before, written = (np.asarray(x, dtype=np.uint32) for x in (mask, before, written))
    if model in ("xor@0", "xor@1", "xor@2"):
        return written ^ mask if elem == int(model[4]) else written
    if model == "stuck0":
        return written & ~mask
    if model == "stuck1":
        return written | mask
    if model == "tf_up":                 # bits that were 0 stay 0
        return written & (before | ~mask)
    if model == "tf_down":               # bits that were 1 stay 1
        return written | (before & mask)
    raise ValueError(model)


def after_write(faults, elem, before, written):
    """cell_after_write for every fault at once: before / written are uint32 arrays in the order of `faults`."""
    stored = np.array(written, dtype=np.uint32, copy=True)
    for model in MODELS:
        sel = np.array([f.model == model for f in faults], dtype=bool)
        if sel.any():
            masks = np.array([f.mask for f in faults], dtype=np.uint32)[sel]
            stored[sel] = cell_after_write(model, masks, elem, np.asarray(before, dtype=np.uint32)[sel], stored[sel])
    return stored


def expected(segment_words, seed: int, inv: int = 0) -> np.ndarray:
    """The words a clean element expects: P (inv = 0) or ~P (inv = 0xFFFFFFFF), segment g keyed with its own seed."""
    return np.concatenate([oprobe.pattern(n, mt.segment_seed(seed, g) ^ inv, base)
                           for g, (n, base) in enumerate(zip(segment_words, np.cumsum([0] + list(segment_words))))])


def march_faulty(segment_words, seed: int, initial, faults=()):
    """The four elements over segments of the given word counts, starting from `initial` (a uint32 or one per word),
    with faulty cells -> one (checksum, mismatches, first_bad, buffer after the element) per element, as
    memtest_oracle.march returns them."""
    n = int(sum(segment_words))
    words = np.array([f.word for f in faults], dtype=np.int64)
    assert words.size == np.unique(words).size and (words.size == 0 or 0 <= words.min() <= words.max() < n), words
    assert all(f.model in MODELS and f.mask & 0xFFFFFFFF for f in faults)
    pattern = expected(segment_words, seed)
    buf = np.broadcast_to(np.asarray(initial, dtype=np.uint32), (n,)).copy()
    out = []
    for k, (reads, writes, inv, delta) in enumerate(mt.MARCH):
        exp = pattern ^ np.uint32(inv)
        cs, bad, first = 0, 0, mt.NO_BAD
        if reads:
            wrong = np.flatnonzero(buf != exp)
            cs, bad, first = oprobe.checksum(buf), int(wrong.size), int(wrong[0]) if wrong.size else mt.NO_BAD
        if writes:
            before = buf[words]
            buf = buf ^ np.uint32(delta) if reads else exp.copy()
            out.append((cs, bad, first, buf.copy()))
            buf[words] = after_write(faults, k, before, buf[words])
        else:
            out.append((cs, bad, first, buf.copy()))
    return out


def pattern_sum(base: int, n: int, seed: int, chunk: int = 1 << 24) -> int:
    """Sum of word(i, seed) over base <= i < base + n, mod 2^64: the pattern summed with numpy in place, fast enough for
    2^32 words (memtest_oracle.range_checksum computes the same with more temporaries)."""
    total = 0
    for start in range(base, base + n, chunk):
        m = min(chunk, base + n - start)
        lo = start & 0xFFFFFFFF
        if lo + m < 1 << 32:
            x = np.arange(lo, lo + m, dtype=np.uint32)
        else:                            # the chunk crosses the wrap of the uint32 index
            x = np.arange(lo, lo + m, dtype=np.uint64).astype(np.uint32)
        x *= np.uint32(oprobe.PATTERN_MUL)
        x ^= np.uint32(seed)
        total += int(x.sum(dtype=np.uint64))
    return total & mt.NO_BAD
