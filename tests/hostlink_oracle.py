"""Oracle of the on-demand host-link self-test (b2dp_hostlink_test), written from its specification rather than from
csrc/hostlink_math.hpp: the store-width schedule of the SM format, the PCIe link capacity, the accepted buffer sizes,
one pass of the SM kernel over a host buffer (with the fault hook) and the verdict.  The pattern, the seed schedule and
the checksum are the probe's (oracle/probe.py)."""
import numpy as np

from oracle import probe as oprobe

DEFAULT_BYTES = 64 << 20
MAX_BYTES = 1 << 30
H2D, D2H, SM = 0, 1, 2
NO_BAD = (1 << 64) - 1
WIDTHS = (16, 8, 4, 2, 1)

# PCIe generation -> (GT/s per lane, payload bits per line bit)
LINE = {1: (2.5, 8 / 10), 2: (5.0, 8 / 10), 3: (8.0, 128 / 130), 4: (16.0, 128 / 130), 5: (32.0, 128 / 130)}


def store_width(vec: int) -> int:
    """Bytes per store for 16-byte vector `vec` of the SM format: 16, 8, 4, 2, 1, then again."""
    return WIDTHS[vec % len(WIDTHS)]


def link_gbs(gen: int, width: int) -> float:
    """Per-direction GB/s of a PCIe link before packet overhead; 0 for an unknown generation or no lanes."""
    if gen not in LINE or width <= 0:
        return 0.0
    gts, eff = LINE[gen]
    return gts * eff * width / 8.0


def buffer_bytes(requested: int) -> int:
    """The bytes per buffer the test uses for a request: 0 = the default, else a multiple of 16 up to 1 GiB; 0 when
    the request is rejected (B2DP_E_INVAL)."""
    if requested == 0:
        return DEFAULT_BYTES
    if requested % 16 or requested > MAX_BYTES:
        return 0
    return requested


def next_seed(seed: int) -> int:
    return oprobe.next_seed(seed)


def sm_pass(src: np.ndarray, seed: int, nxt: int, fault_word: int = 0, fault_mask: int = 0):
    """One pass of the SM kernel over a host buffer: the fault hook flips fault_word as it is read, every word is
    checked against pattern(seed) and re-keyed to nxt.  Returns (checksum, mismatches, first_bad, dst)."""
    seen = src.copy()
    if fault_mask:
        seen[fault_word] ^= np.uint32(fault_mask)
    return oprobe.probe_pass(seen, seed, nxt)


def check(buf: np.ndarray, seed: int):
    """The host's check of a destination buffer: (wrong words, first wrong index or NO_BAD)."""
    bad = np.nonzero(buf != oprobe.pattern(len(buf), seed))[0]
    return len(bad), (int(bad[0]) if len(bad) else NO_BAD)


def healthy(calls_ok: bool, seq_ok: bool, checksums_ok: bool, rounds, mismatches) -> bool:
    return bool(calls_ok and seq_ok and checksums_ok and all(r >= 1 for r in rounds)
                and all(m == 0 for m in mismatches))
