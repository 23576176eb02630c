"""hbm_probe_queue, the health probe's kernel, launched directly (tests/native/probe_queue_kernels.cu) against the
exact uint64 arithmetic of oracle/probe.py: checksum, mismatch count, first bad word, the whole written buffer, a
guard region past it and the control block, tile queue included, at the launch shapes and faults of
tests/probe_cases.py.  Run with -m gpu on an H100."""
import itertools

import numpy as np
import pytest

import probe_cases as pc
from oracle import probe as oprobe
from probe_queue_kernels import QUEUE

pytestmark = pytest.mark.gpu

GUARD_WORDS = 64                    # words past n_vec that no launch may touch
SENTINEL = 0x5A5A5A5A
# (checksum, mismatches, first_bad, t_start_ns, done, next_tile): what the last CTA and the last claim leave behind
RESET_CTL = (0, 0, oprobe.NO_BAD, oprobe.NO_BAD, 0, 0)
_SEQ = itertools.count(1)


@pytest.fixture(scope="module")
def H():
    import probe_queue_kernels
    assert probe_queue_kernels.variant() == QUEUE
    h = probe_queue_kernels.Harness(0)
    yield h
    h.close()


def _dev(words: np.ndarray, extra=GUARD_WORDS):
    """A device copy of a uint32 buffer followed by `extra` sentinel words."""
    import torch
    host = np.full(words.size + extra, SENTINEL, dtype=np.uint32)
    host[:words.size] = words
    return torch.from_numpy(host.view(np.int32)).to("cuda:0")


def _host(t):
    return t.cpu().numpy().view(np.uint32)


def _ctl(H):
    c = H.read_ctl()
    return (c.checksum, c.mismatches, c.first_bad, c.t_start_ns, c.done, c.pad)   # pad = ProbeCtl::next_tile


def test_queue_kernel_equals_oracle_on_every_case(H):
    """One control block for all cases, in order: grids and sizes change from launch to launch, so a queue the last
    claim failed to reset (or a counter the last CTA failed to reset) shows up in the next case and in the block."""
    import torch
    for case in pc.cases(QUEUE, QUEUE.product_grid(H.sms)):
        src = case.src()
        d_src = _dev(src)
        d_dst = _dev(np.empty(0, dtype=np.uint32), case.n_words + GUARD_WORDS)
        torch.cuda.synchronize()
        seq = next(_SEQ)
        r = H.run(d_src, d_dst, case.n_vec, case.seed, case.delta, case.grid, seq)
        cs, bad, first, want_dst = oprobe.probe_pass(src, case.seed, case.seed ^ case.delta)
        got = (r.checksum, r.mismatches, r.first_bad)
        assert got == (cs, bad, first), (case.name, got, (cs, bad, first))
        assert r.seq == seq and 0 < r.t_start_ns <= r.t_end_ns, (case.name, r.seq, r.t_start_ns, r.t_end_ns)
        out = _host(d_dst)
        if not np.array_equal(out[:case.n_words], want_dst):
            wrong = np.nonzero(out[:case.n_words] != want_dst)[0]
            raise AssertionError("%s: %d dst words differ, first at %d: %#x != %#x"
                                 % (case.name, wrong.size, wrong[0], out[wrong[0]], want_dst[wrong[0]]))
        assert (out[case.n_words:] == SENTINEL).all(), (case.name, "write past n_vec")
        assert (_host(d_src) == np.concatenate([src, np.full(GUARD_WORDS, SENTINEL, np.uint32)])).all(), case.name
        assert _ctl(H) == RESET_CTL, (case.name, _ctl(H))


@pytest.mark.parametrize("grid", [1, 2, 5, 264, 1000])
def test_queue_hands_out_every_tile_once_at_any_grid(H, grid):
    """Back-to-back launches on one stream at one grid: each pass must re-key every tile exactly once (a tile taken
    twice or never shows in the buffer), and the queue must start from 0 for the next pass."""
    import torch
    n_vec = 37 * QUEUE.vec_per_tile + 3
    seed = 0x5EED1234
    a = _dev(oprobe.pattern(4 * n_vec, seed))
    b = _dev(np.empty(0, dtype=np.uint32), 4 * n_vec + GUARD_WORDS)
    torch.cuda.synchronize()
    for _ in range(4):
        nxt = oprobe.next_seed(seed)
        seq = next(_SEQ)
        r = H.run(a, b, n_vec, seed, seed ^ nxt, grid, seq)
        assert (r.mismatches, r.first_bad) == (0, oprobe.NO_BAD)
        assert r.checksum == oprobe.expected_checksum(4 * n_vec, seed)
        assert np.array_equal(_host(b)[:4 * n_vec], oprobe.pattern(4 * n_vec, nxt))
        assert _ctl(H) == RESET_CTL
        a, b, seed = b, a, nxt


def test_harness_refuses_out_of_bounds_and_misaligned_launches(H):
    import probe_queue_kernels as pq
    import torch
    a = torch.zeros(4096, dtype=torch.int32, device="cuda:0")
    b = torch.zeros(4096, dtype=torch.int32, device="cuda:0")
    torch.cuda.synchronize()
    assert H.run_rc(a, b, 1025, 1, 0, 0, 1)[0] == pq.E_SIZE
    assert H.run_rc(a, b[:2048], 1024, 1, 0, 0, 1)[0] == pq.E_SIZE
    assert H.run_rc(a[4:], b, 16, 1, 0, 0, 1)[0] == pq.E_ALIGN
    assert H.run_rc(a, b[4:], 16, 1, 0, 0, 1)[0] == pq.E_ALIGN
    assert H.run_rc(a, b, 16, 1, 0, -1, 1)[0] == pq.E_GRID
    assert H.run_rc(a, b, 16, 1, 0, (1 << 20) + 1, 1)[0] == pq.E_GRID
    assert (b == 0).all() and _ctl(H) == RESET_CTL


def test_product_shape_reaches_its_resident_ctas(H):
    """The product grid is SMs x 2: two CTAs must fit on one SM at once with the launch's real shared memory
    (6 x 8 KiB ring = 96 KiB staged per SM, as the former probe kernel)."""
    assert H.occupancy() >= QUEUE.ctas_per_sm


def test_counters_past_32_bits(H):
    """2^32 + 2^22 words of 0xFFFFFFFF through the queue kernel at the product grid: the checksum carries past 2^64
    and the mismatch count passes 2^32.  word(i, seed) == 0xFFFFFFFF exactly at i = ~seed * K^-1 (mod 2^32), once
    per 2^32-word period, so the count and the first bad word follow from that index."""
    import torch
    n_words = (1 << 32) + (1 << 22)
    n_vec = n_words // 4
    free, _ = torch.cuda.mem_get_info(0)
    if free < 2 * n_words * 4 + (2 << 30):
        pytest.skip("not enough free HBM for two %.1f GiB buffers" % (n_words * 4 / 2 ** 30))
    k_inv = pow(oprobe.PATTERN_MUL, -1, 1 << 32)
    src = torch.full((n_words,), -1, dtype=torch.int32, device="cuda:0")
    dst = torch.empty(n_words, dtype=torch.int32, device="cuda:0")
    try:
        seed0 = oprobe.initial_seed(0)
        for seed, delta in ((seed0, seed0 ^ oprobe.next_seed(seed0)), (0xFFFFFFFF, 0)):
            i0 = ((~seed & 0xFFFFFFFF) * k_inv) & 0xFFFFFFFF
            assert oprobe.pattern(1, seed, i0)[0] == 0xFFFFFFFF
            matches = 1 + (i0 < (1 << 22))
            torch.cuda.synchronize()
            seq = next(_SEQ)
            r = H.run(src, dst, n_vec, seed, delta, 0, seq)
            assert r.checksum == (n_words * 0xFFFFFFFF) & oprobe.NO_BAD
            assert r.mismatches == n_words - matches and r.mismatches > 1 << 32
            assert r.first_bad == (1 if i0 == 0 else 0)
            want = np.uint32(0xFFFFFFFF ^ delta).view(np.int32).item()
            assert all(bool((part == want).all()) for part in dst.split(1 << 28))
            assert _ctl(H) == RESET_CTL
    finally:
        del src, dst
        torch.cuda.empty_cache()
