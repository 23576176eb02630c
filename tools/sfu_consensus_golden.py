"""Capture the SFU self-test's reference words on an H100 as golden values.

Runs the reference launch (one CTA on every SM) of every format at two fixed seeds through
tests/native/libsfu_test_kernels_test.so, requires every SM to agree bit for bit, and writes the SHA-256 of each
(seed, format, tile)'s [thread][word] words to a JSON file (default tests/golden/sfu_sm90_consensus.json), together with
the card's name and power limit.  tests/test_gpu_sfu_test.py compares later runs with that file.

    python tools/sfu_consensus_golden.py [out.json]
"""
import hashlib
import json
import os
import subprocess
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))

import sfu_test_oracle as so  # noqa: E402
from test_gpu_sfu_test import Harness  # noqa: E402

SEEDS = [0x5F0, 0xC0FFEE17]


def main():
    out = sys.argv[1] if len(sys.argv) > 1 else os.path.join(ROOT, "tests", "golden", "sfu_sm90_consensus.json")
    card = subprocess.run(["nvidia-smi", "-i", "0", "--query-gpu=name,power.limit,driver_version", "--format=csv,noheader"],
                          capture_output=True, text=True).stdout.strip()
    h = Harness(0)
    sha = {}
    try:
        for seed in SEEDS:
            for fmt in so.FORMATS:
                d, recs, _ = h.dump(fmt, seed)
                assert all(r.seq == 7 for r in recs) and (d == d[0][None]).all(), "the SMs disagree"
                for t in range(so.TILES):
                    sha["%d/%s/%d" % (seed, so.NAMES[fmt], t)] = hashlib.sha256(d[0][t].tobytes()).hexdigest()
    finally:
        h.close()
    with open(out, "w") as f:
        json.dump({"card": card, "sms": h.sms, "seeds": SEEDS, "sha256": sha}, f, indent=1, sort_keys=True)
        f.write("\n")
    print("wrote %d digests for %s to %s" % (len(sha), card, out))


if __name__ == "__main__":
    main()
