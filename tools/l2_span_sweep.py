#!/usr/bin/env python3
"""Sweep the L2 self-test's L2_WORD march over spans from 1 MiB to 4 x cudaDevAttrL2CacheSize and print TB/s per span.

Runs the kernel through the test harness (tests/native/libl2_test_kernels_test.so, built by __graft_entry__.build()),
cooperatively on every resident CTA, for --ms per span.  The rate is the march's bytes read and written (10 x span per
comparison) over the launch's CUDA-event time; it falls where the span stops fitting in what the L2 keeps resident for
every SM, and the default span (3/8 of the L2) must sit below that knee.  Prints the card, its power limit and maximum
SM clock first.  Usage: python tools/l2_span_sweep.py [--ms 300] [--out profiles/l2_span_sweep_h100.txt]
"""
import argparse
import os
import subprocess
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, os.path.join(ROOT, "tests"))

from test_gpu_l2_test import Harness  # noqa: E402
import l2_test_oracle as lo  # noqa: E402


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--ms", type=float, default=300)
    ap.add_argument("--out", default=None)
    a = ap.parse_args()
    lines = []
    smi = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                         stdout=subprocess.PIPE, stderr=subprocess.STDOUT, text=True).stdout.strip()
    H = Harness(0)
    try:
        grid = H.sms * H.occupancy(lo.WORD)
        lines.append("card: %s; L2 %d KiB; %d CTAs; %g ms per span" % (smi, H.l2 >> 10, grid, a.ms))
        lines.append("%10s %6s %10s %8s" % ("span_MiB", "K", "span/L2", "TB/s"))
        unit = grid * lo.BLOCK_WORDS * 4
        spans = sorted({max(1, (m << 20) // unit) for m in (1, 2, 4, 8, 12, 16, 20, 24, 28, 32, 40, 48)} |
                       {max(1, H.l2 * f // 8 // unit) for f in (2, 3, 4, 5, 6, 8, 12, 16, 24, 32)})
        for K in spans:
            recs, ms, k, _ = H.run(lo.WORD, 0x5EED + K, a.ms, K=K)
            span = k * unit
            tbs = 10 * span * recs[0].comparisons / (ms * 1e-3) / 1e12
            bad = sum(r.mismatches for r in recs)
            lines.append("%10.2f %6d %10.3f %8.2f%s" % (span / (1 << 20), k, span / H.l2, tbs,
                                                        "  MISMATCHES %d" % bad if bad else ""))
            print(lines[-1], flush=True)
    finally:
        H.close()
    text = "\n".join(lines) + "\n"
    print(text)
    if a.out:
        os.makedirs(os.path.dirname(os.path.abspath(a.out)), exist_ok=True)
        with open(a.out, "w") as f:
            f.write(text)


if __name__ == "__main__":
    main()
