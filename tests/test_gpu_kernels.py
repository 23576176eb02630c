"""The HBM probe kernels of hbm_probe.cuh launched directly (tests/native/probe_kernels.cu), every instantiation the
product or tools/probe_sweep uses, against the exact uint64 arithmetic of oracle/probe.py: checksum, mismatch count,
first bad word and the whole written buffer, at the launch shapes and faults of tests/probe_cases.py.  Run with -m gpu
on an H100."""
import itertools

import numpy as np
import pytest

import probe_cases as pc
from oracle import probe as oprobe

pytestmark = pytest.mark.gpu

GUARD_WORDS = 64                    # words past n_vec that no launch may touch
SENTINEL = 0x5A5A5A5A
RESET_CTL = (0, 0, oprobe.NO_BAD, oprobe.NO_BAD, 0)
VARIANT_INDEX = {v.name: i for i, v in enumerate(pc.VARIANTS)}
_SEQ = itertools.count(1)           # every launch in this module gets its own sequence number


@pytest.fixture(scope="module")
def H():
    import probe_kernels
    assert probe_kernels.variants() == list(pc.VARIANTS)
    h = probe_kernels.Harness(0)
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
    return (c.checksum, c.mismatches, c.first_bad, c.t_start_ns, c.done)


@pytest.mark.parametrize("name", [v.name for v in pc.VARIANTS])
def test_kernel_equals_oracle_on_every_case(H, name):
    """One control block for all cases, in order: grids and sizes change from launch to launch, so a counter the last
    CTA failed to reset shows up in the next case's result and in the control block itself."""
    import torch
    vi = VARIANT_INDEX[name]
    v = pc.VARIANTS[vi]
    for case in pc.cases(v, v.product_grid(H.sms)):
        src = case.src()
        d_src = _dev(src)
        d_dst = _dev(np.empty(0, dtype=np.uint32), case.n_words + GUARD_WORDS)
        torch.cuda.synchronize()
        seq = next(_SEQ)
        r = H.run(vi, d_src, d_dst, case.n_vec, case.seed, case.delta, case.grid, seq)
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


@pytest.mark.parametrize("n_vec", [0, 1, 3, 255, 256 * 132 * 8 - 1, 256 * 132 * 8 + 1, (1 << 20) + 5])
def test_fill_equals_pattern(H, n_vec):
    import torch
    seed = 0xC0FFEE ^ n_vec
    d = _dev(np.empty(0, dtype=np.uint32), 4 * n_vec + GUARD_WORDS)
    torch.cuda.synchronize()
    H.fill(d, n_vec, seed)
    out = _host(d)
    assert np.array_equal(out[:4 * n_vec], oprobe.pattern(4 * n_vec, seed))
    assert (out[4 * n_vec:] == SENTINEL).all()


def test_harness_refuses_out_of_bounds_and_misaligned_launches(H):
    import probe_kernels
    import torch
    a = torch.zeros(4096, dtype=torch.int32, device="cuda:0")
    b = torch.zeros(4096, dtype=torch.int32, device="cuda:0")
    torch.cuda.synchronize()
    assert H.run_rc(0, a, b, 1025, 1, 0, 0, 1)[0] == probe_kernels.E_SIZE
    assert H.run_rc(0, a, b[:2048], 1024, 1, 0, 0, 1)[0] == probe_kernels.E_SIZE
    assert H.run_rc(0, a[4:], b, 16, 1, 0, 0, 1)[0] == probe_kernels.E_ALIGN
    assert H.run_rc(0, a, b[4:], 16, 1, 0, 0, 1)[0] == probe_kernels.E_ALIGN
    assert H.run_rc(len(pc.VARIANTS), a, b, 16, 1, 0, 0, 1)[0] == probe_kernels.E_VARIANT
    assert (b == 0).all() and _ctl(H) == RESET_CTL
    with pytest.raises(RuntimeError):
        H.fill(b, 1025, 1)


def test_product_shapes_reach_their_resident_ctas(H):
    """The product grid is SMs x 2 for both product kernels: two CTAs of each must fit on one SM at once with the
    launch's real shared memory (96 KiB staged per SM for the TMA ring, DESIGN.md 4.1)."""
    for name in ("tma_4_1024_3", "r128_512_2"):
        vi = VARIANT_INDEX[name]
        assert H.occupancy(vi) >= pc.VARIANTS[vi].ctas_per_sm, name
    for vi, v in enumerate(pc.VARIANTS):
        assert H.occupancy(vi) >= 1, v.name


def test_counters_past_32_bits(H):
    """2^32 + 2^22 words of 0xFFFFFFFF through the product TMA kernel: the checksum carries past 2^64 and the mismatch
    count passes 2^32.  word(i, seed) == 0xFFFFFFFF exactly at i = ~seed * K^-1 (mod 2^32), once per 2^32-word
    period, so the count and the first bad word follow from that index."""
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
        # seed 0xFFFFFFFF puts the matching index at i0 = 0: words 0 and 2^32 match, the first bad word is 1
        seed0 = oprobe.initial_seed(0)
        for seed, delta in ((seed0, seed0 ^ oprobe.next_seed(seed0)), (0xFFFFFFFF, 0)):
            i0 = ((~seed & 0xFFFFFFFF) * k_inv) & 0xFFFFFFFF
            assert oprobe.pattern(1, seed, i0)[0] == 0xFFFFFFFF
            matches = 1 + (i0 < (1 << 22))
            torch.cuda.synchronize()
            seq = next(_SEQ)
            r = H.run(0, src, dst, n_vec, seed, delta, 0, seq)
            assert r.checksum == (n_words * 0xFFFFFFFF) & oprobe.NO_BAD
            assert r.mismatches == n_words - matches and r.mismatches > 1 << 32
            assert r.first_bad == (1 if i0 == 0 else 0)
            want = np.uint32(0xFFFFFFFF ^ delta).view(np.int32).item()
            assert all(bool((part == want).all()) for part in dst.split(1 << 28))
            assert _ctl(H) == RESET_CTL
    finally:
        del src, dst
        torch.cuda.empty_cache()
