#!/usr/bin/env python3
"""Sweep the L1 self-test's L1_DATA format over per-SM spans from one 2 KiB block per CTA to about 1 MiB, at
shared-memory carve-outs of 0 and 100, and print TB/s per span; then L1_TEX (its image is a fixed 128 KiB) at both
carve-outs.

Runs the kernel through the test harness (tests/native/libl1_test_kernels_test.so, built by __graft_entry__.build())
on every resident CTA, for --ms per point.  A span is a whole number K of 2 KiB blocks per CTA, so the per-SM spans are
multiples of 2 KiB x the CTAs per SM (10 KiB at 5 CTAs): each target of 16 KiB .. 1 MiB is rounded down to one, and the
output lists the spans actually run.  The rate is the bytes the loads deliver (L1_DATA: and its stores) over the
launch's CUDA-event time.  It falls where the span stops fitting in what L1 keeps for every SM; the default span
(128 KiB per SM) must sit below that fall at carve-out 0.  Prints the card, its power limit and maximum SM clock first.
Usage: python tools/l1_span_sweep.py [--ms 200] [--out profiles/l1_span_sweep_h100.txt]
"""
import argparse
import os
import subprocess
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, os.path.join(ROOT, "tests"))

from test_gpu_l1_test import Harness  # noqa: E402
import l1_test_oracle as lo  # noqa: E402

BLOCK_BYTES = lo.BLOCK * 4


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--ms", type=float, default=200)
    ap.add_argument("--out", default=None)
    a = ap.parse_args()
    lines = []
    smi = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                         stdout=subprocess.PIPE, stderr=subprocess.STDOUT, text=True).stdout.strip()
    H = Harness(0)
    try:
        occ = H.occupancy(lo.DATA)
        lines.append("card: %s; %d SMs; L1_DATA %d CTAs per SM; %g ms per point" % (smi, H.sms, occ, a.ms))
        lines.append("%8s %12s %6s %8s %8s" % ("format", "carveout_%", "K", "KiB/SM", "TB/s"))
        spans = sorted({max(1, (kib << 10) // (occ * BLOCK_BYTES))
                        for kib in (16, 32, 48, 64, 96, 128, 160, 192, 224, 256, 320, 384, 512, 768, 1024)})
        for carve in (0, 100):
            for K in spans:
                recs, ms, k, _ = H.run(lo.DATA, 0x5EED + K, a.ms, K=K, carveout=carve)
                per_cta = 4 * k * BLOCK_BYTES            # one write and three read passes per comparison
                tbs = per_cta * sum(r.comparisons for r in recs) / (ms * 1e-3) / 1e12
                bad = sum(r.mismatches for r in recs)
                lines.append("%8s %12d %6d %8d %8.2f%s" % ("data", carve, k, k * BLOCK_BYTES * occ >> 10, tbs,
                                                          "  MISMATCHES %d" % bad if bad else ""))
                print(lines[-1], flush=True)
            recs, ms, _, _ = H.run(lo.TEX, 0x5EED, a.ms, carveout=carve)
            per_cta = lo.THREADS * lo.STEPS * 8 * 16      # eight 16-byte fetches per thread and step
            tbs = per_cta * sum(r.comparisons for r in recs) / (ms * 1e-3) / 1e12
            bad = sum(r.mismatches for r in recs)
            lines.append("%8s %12d %6s %8d %8.2f%s" % ("tex", carve, "-", lo.TEXELS * 16 >> 10, tbs,
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
