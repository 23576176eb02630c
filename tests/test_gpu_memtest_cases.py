"""The memory-test march (hbm_march_tma, csrc/hbm_memtest.cuh) on a real H100 against the faulty-memory oracle
(tests/memtest_faults.py), through the test-only harness tests/native/libmemtest_kernels_test.so.

- Every case of tests/memtest_cases.py: the elements run one launch at a time, and after each writing launch the
  faulty words are read back and given what memtest_faults.cell_after_write says the faulty cell holds, so the GPU and
  the oracle can only disagree because of the kernel.  After each element: the result block, the whole buffer, the
  guard region past each segment, the control block's reset, seq and the timestamps.  The segments are carved out of
  one allocation in an order that is not the table's.
- Past 2^32 words, at the kernel: 16 segments of 1 GiB and one of 4 tiles (2^32 + 16,384 words).  Sums from numpy,
  windows at both ends of every segment and across the wrap, a flip at word 2^32 + 5, and elements run out of order so
  the mismatch count passes 2^32.
- Past 2^32 words, through the ABI: a 17 GiB b2dp_memtest is healthy, so the host's closed-form checksum equals the
  kernel's sums across the wrap; a fault at word 2^32 + 5 is reported there and latched until probe_reset.

The machines are shared: this file's largest allocation is about 17 GiB (the 2^32-word march, or the 17 GiB memtest),
one at a time, and each test frees its memory before the next.  Run with -m gpu."""
import os

import numpy as np
import pytest

import memtest_cases as mc
import memtest_faults as mf
import memtest_oracle as mt
from oracle import probe as oprobe
from test_gpu_memtest import GUARD_WORDS, LIB_PATH, Harness

pytestmark = pytest.mark.gpu

GiB = 1 << 30
WRAP = 1 << 32
RESET_CTL = (0, 0, mt.NO_BAD, mt.NO_BAD, 0)
SENTINEL_I32 = np.uint32(mc.SENTINEL).view(np.int32).item()


@pytest.fixture(scope="module")
def H():
    if not os.path.exists(LIB_PATH):
        pytest.skip("run __graft_entry__.build() first")
    h = Harness(0)
    yield h
    h.close()


@pytest.fixture(scope="module")
def on_this_part(H):
    return {c.name: c for c in mc.cases(2 * H.sms)}


def _u32(t):
    return t.cpu().numpy().view(np.uint32)


def _element(H, ptrs, sizes, seed, k, grid):
    """One launch, with the checks every launch gets: seq, timestamps and the control block's reset."""
    import torch
    torch.cuda.synchronize()                       # the harness launches on a stream of its own
    r = H.element(ptrs, sizes, seed, k, grid)
    assert r.seq == H.seq and 0 < r.t_start_ns <= r.t_end_ns, (k, r.seq, r.t_start_ns, r.t_end_ns)
    c = H.ctl(k)
    assert (c.checksum, c.mismatches, c.first_bad, c.t_start_ns, c.done) == RESET_CTL, k
    return r


@pytest.mark.parametrize("name", [c.name for c in mc.cases()])
def test_march_kernel_matches_the_faulty_memory_oracle(H, on_this_part, name):
    import torch
    c = on_this_part[name]
    words = c.seg_words
    slot = words[0] + GUARD_WORDS
    mem = torch.full((len(words) * slot,), SENTINEL_I32, dtype=torch.int32, device="cuda:0")
    off = [slot * s for s in c.slots]                            # segment g starts at word off[g] of mem
    ptrs, sizes = [mem.data_ptr() + 4 * o for o in off], [4 * w for w in words]
    table = np.concatenate([np.arange(o, o + w) for o, w in zip(off, words)])   # mem index of each table word
    guard = np.ones(mem.numel(), dtype=bool)
    guard[table] = False
    at_np = table[np.array([f.word for f in c.faults], dtype=np.int64)]
    at = torch.from_numpy(at_np).to("cuda:0")
    want = c.march()
    for k in range(4):
        writes = mt.MARCH[k][1]
        if c.faults and writes:
            before = _u32(mem[at])
        r = _element(H, ptrs, sizes, c.seed, k, c.grid)
        cs, mm, fb, buf = want[k]
        assert (r.checksum, r.mismatches, r.first_bad) == (cs, mm, fb), (name, k)
        got = _u32(mem)
        assert np.array_equal(got[table], buf), (name, k, np.flatnonzero(got[table] != buf)[:8])
        assert np.all(got[guard] == mc.SENTINEL), (name, k, "guard region written")
        if c.faults and writes:                                  # the faulty cells act on what the kernel wrote
            stored = mf.after_write(c.faults, k, before, got[at_np])
            mem[at] = torch.from_numpy(stored.view(np.int32)).to("cuda:0")


# ---- past 2^32 words ---------------------------------------------------------------------------------------------------
def test_march_kernel_past_2_32_words(H):
    """2^32 + 16,384 words: the uint32 pattern index wraps at the start of the last segment, first_bad carries the high
    bits, mismatch counts pass 2^32, and the sums equal the pattern summed in numpy.  Only windows are copied back."""
    import torch
    seg_words = [1 << 28] * 16 + [4 * mc.TILE_WORDS]
    n = sum(seg_words)
    assert n == WRAP + 16384
    if torch.cuda.mem_get_info(0)[0] < 20 * GiB:
        pytest.skip("needs 16 GiB + 4 GiB of free HBM")
    seed = 0x0DDC0FFE
    starts = np.cumsum([0] + seg_words)
    seeds = [mt.segment_seed(seed, g) for g in range(len(seg_words))]
    sum_p = sum(mf.pattern_sum(int(starts[g]), w, seeds[g]) for g, w in enumerate(seg_words)) & mt.NO_BAD
    sum_not_p = (n * 0xFFFFFFFF - sum_p) & mt.NO_BAD
    segs = [torch.empty(w + GUARD_WORDS, dtype=torch.int32, device="cuda:0") for w in seg_words]
    try:
        for s, w in zip(segs, seg_words):
            s[w:] = SENTINEL_I32
        ptrs, sizes = [s.data_ptr() for s in segs], [4 * w for w in seg_words]
        win = 4096

        def windows(inv):
            for g, (s, w) in enumerate(zip(segs, seg_words)):
                for lo in (0, w - win):
                    got = _u32(s[lo:lo + win])
                    assert np.array_equal(got, oprobe.pattern(win, seeds[g] ^ inv, int(starts[g]) + lo)), (g, lo, inv)
                assert np.all(_u32(s[w:]) == mc.SENTINEL), (g, "guard region written")
            past = _u32(segs[16][:win])                          # words 2^32 ...: segment 16's seed, not segment 0's
            assert not np.array_equal(past, oprobe.pattern(win, seeds[0] ^ inv, WRAP))

        def run(k):
            return _element(H, ptrs, sizes, seed, k, 0)

        # a clean march
        r = run(0)
        assert (r.checksum, r.mismatches, r.first_bad) == (0, 0, mt.NO_BAD)
        windows(0)
        for k, total, inv in ((1, sum_p, mt.INV), (2, sum_not_p, 0), (3, sum_p, 0)):
            r = run(k)
            assert (r.checksum, r.mismatches, r.first_bad) == (total, 0, mt.NO_BAD), k
            windows(inv)

        # one flip past the wrap, after E0
        word, mask = WRAP + 5, 0x80
        run(0)
        v = int(segs[16][5].item()) & 0xFFFFFFFF
        p = int(oprobe.pattern(1, seeds[16], word)[0])
        assert v == p
        segs[16][5] = np.uint32(v ^ mask).view(np.int32).item()
        for k, total, read, good in ((1, sum_p, p ^ mask, p), (2, sum_not_p, ~(p ^ mask), ~p), (3, sum_p, p ^ mask, p)):
            r = run(k)
            cs = (total - (good & 0xFFFFFFFF) + (read & 0xFFFFFFFF)) & mt.NO_BAD
            assert (r.checksum, r.mismatches, r.first_bad) == (cs, 1, word), k

        # out of order: E2 and E3 after E0 expect the other pattern in every word
        run(0)
        r = run(2)
        assert (r.checksum, r.mismatches, r.first_bad) == (sum_p, n, 0)
        windows(mt.INV)
        r = run(3)
        assert (r.checksum, r.mismatches, r.first_bad) == (sum_not_p, n, 0)
        assert r.mismatches > WRAP
    finally:
        del segs
        torch.cuda.empty_cache()


def test_memtest_past_2_32_words_through_the_abi(pkg):
    """b2dp_memtest over 17 GiB (17 segments, 4.56e9 words): healthy means every reading element summed to the host's
    closed form (memtest_expected_checksum) across the wrap; a flip at word 2^32 + 5 is found there and latched."""
    import torch
    torch.cuda.init()
    max_bytes = 17 * GiB
    with pkg.Context("cuda:devices=0,bytes=%d,calib=1" % (64 << 20)) as ctx:
        free, total = torch.cuda.mem_get_info(0)
        if sum(mt.plan(free, total, 0, max_bytes)) < max_bytes:
            pytest.skip("the memory test's plan does not reach 17 GiB (free %.1f GiB)" % (free / GiB))
        (r,) = ctx.memtest(0, max_bytes=max_bytes)
        assert r.healthy and r.err == 0, r
        assert r.n_segments == 17 and r.bytes_tested == max_bytes
        assert r.mismatches == [0, 0, 0, 0] and r.first_bad_word == mt.NO_BAD
        (r,) = ctx.memtest(0, max_bytes=max_bytes, fault_word=WRAP + 5, fault_mask=0x80)
        assert r.bytes_tested == max_bytes and r.err == 0, r
        assert r.mismatches == [0, 1, 1, 1] and r.first_bad_word == WRAP + 5 and not r.healthy
        (p,) = ctx.probe_health(min_gbs=1e-3)
        assert p.flags & pkg._native.RES_MEMTEST and not p.healthy
        ctx.probe_reset(0)
        (p,) = ctx.probe_health(min_gbs=1e-3)
        assert p.healthy and not p.flags & pkg._native.RES_MEMTEST
