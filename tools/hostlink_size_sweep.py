#!/usr/bin/env python3
"""Sweep the host-link self-test over buffer sizes from 1 MiB to 1 GiB and print GB/s per format.

Runs b2dp_hostlink_test on device 0 through the library (built by __graft_entry__.build()), --ms per format and size.
H2D and D2H are bytes x rounds over the summed CUDA-event time of the copies in that direction; SM is the bytes the SMs
read plus the bytes they wrote over the kernels' event time.  Each row also carries the PCIe generation and width NVML
reported while transfers were in flight.  The default buffer (64 MiB) must sit on the plateau of the copy rates.
Prints the card and its power limit first.  Usage: python tools/hostlink_size_sweep.py [--ms 500] [--out FILE]
"""
import argparse
import importlib
import os
import subprocess
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

MiB = 1 << 20


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--ms", type=int, default=500)
    ap.add_argument("--out", default=None)
    a = ap.parse_args()
    pkg = importlib.import_module("k8s-device-plugin_b200")
    smi = subprocess.run(["nvidia-smi", "-i", "0", "--query-gpu=name,power.limit", "--format=csv,noheader"],
                         stdout=subprocess.PIPE, stderr=subprocess.STDOUT, text=True).stdout.strip()
    lines = ["card: %s; %d ms per format and size" % (smi, a.ms),
             "%9s %7s %7s %7s %9s %8s %6s %9s %s" % ("bytes_MiB", "h2d", "d2h", "sm", "rounds", "link", "numa",
                                                     "link_GB/s", "verdict")]
    print(lines[0])
    print(lines[1], flush=True)
    with pkg.Context("cuda:devices=0,bytes=%d,calib=1" % (64 * MiB)) as ctx:
        ctx.hostlink_test(0, bytes=MiB, duration_ms=20)          # the first launch loads the kernels
        for mib in (1, 2, 4, 8, 16, 32, 64, 128, 256, 512, 1024):
            (r,) = ctx.hostlink_test(0, bytes=mib * MiB, duration_ms=a.ms, even_if_busy=True)
            lines.append("%9d %7.2f %7.2f %7.2f %9s %8s %6d %9.1f %s" % (
                mib, r.gbs[0], r.gbs[1], r.gbs[2], "/".join(str(k) for k in r.rounds),
                "gen%dx%d" % (r.link_gen, r.link_width), r.host_numa_node, r.link_gbs,
                "Healthy" if r.healthy else "UNHEALTHY flags 0x%x err %d" % (r.flags, r.err)))
            print(lines[-1], flush=True)
            if not r.healthy:
                ctx.probe_reset(0)
    text = "\n".join(lines) + "\n"
    if a.out:
        os.makedirs(os.path.dirname(os.path.abspath(a.out)), exist_ok=True)
        with open(a.out, "w") as f:
            f.write(text)


if __name__ == "__main__":
    main()
