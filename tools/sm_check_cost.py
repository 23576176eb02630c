"""What the heartbeat's SM check (cuda: sm_check=<ms>) costs on one H100, measured in one run next to the card's name,
power limit and maximum SM clock.

1. The HBM pass with and without the slice: tools/b200dp_cli <uri> cycle 40 [idle_ms] for `cuda:` and
   `cuda:sm_check=10`, back to back and with a 1,000 ms idle gap, alternating, twice.  These run before this process
   opens a context of its own, which would make the GPU busy for the CLI (another process uses it) and skip its slices.
2. Per suite, at sm_check=10 and sm_check=100: the slice's kernel time per format (the event time between its launches,
   b2dp_compute_test_result.ms), its wall time on the GPU's worker (table build, allocations, the SFU reference step,
   the L1 bind, the launches and the release), and the difference, which is the setup; and the probe_health call.
   Each value is the median over three rotations after one warm-up rotation.  Every slice's SM coverage is recorded.
3. Per pass in this process, probe_health back to back and after 1,000 ms idle: the pass's frac (its rate over the
   calibrated ceiling) by the suite whose slice ran just before it, and every RES_SLOW.

Prints the report; --out also writes it to a file.
Usage: python tools/sm_check_cost.py [--out profiles/sm_check_cost_h100.txt]"""
import argparse
import importlib
import json
import os
import re
import statistics
import subprocess
import sys
import time

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
CLI = os.path.join(ROOT, "tools", "b200dp_cli")
LINE = re.compile(r"^(\S+) SM check (.+?): (Healthy|Unhealthy \(latched\)), SMs (\d+)/(\d+), mismatches \S+ "
                  r"(\d+)/(\d+)/(\d+), ([\d.]+)/([\d.]+)/([\d.]+) ms, ([\d.]+) ms on the worker(.*)$")
SUITES = ["compute test", "FP test", "SFU test", "shared-memory test", "register-file test", "integer test",
          "L2 test", "half-precision test", "sync test", "L1 test"]


def card():
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader", "-i", "0"],
                       capture_output=True, text=True)
    return q.stdout.strip() or "nvidia-smi gave nothing: %s" % q.stderr.strip()


def slice_costs(pkg, ms, out):
    N = pkg._native
    logs = []
    N.set_log_callback(lambda level, msg: logs.append(msg))
    rows = {s: {"kernel": [], "wall": [], "call": [], "sms": set(), "healthy": True} for s in SUITES}
    try:
        with pkg.Context("cuda:devices=0,sm_check=%d" % ms) as ctx:
            for _ in range(10):                                   # warm-up rotation: loads every suite's kernels
                ctx.probe_health(timed=False)
            for _ in range(30):
                del logs[:]
                t0 = time.perf_counter()
                (p,) = ctx.probe_health(timed=False)
                call = (time.perf_counter() - t0) * 1e3
                m = [LINE.match(x) for x in logs]
                m = [x for x in m if x]
                if len(m) != 1:
                    out.append("  pass without exactly one SM check line: flags=0x%x sm_check=%d" % (p.flags, p.sm_check))
                    continue
                m = m[0]
                r = rows[m.group(2)]
                kern = [float(m.group(i)) for i in (9, 10, 11)]
                r["kernel"].append(kern)
                r["wall"].append(float(m.group(12)))
                r["call"].append(call)
                r["sms"].add("%s/%s" % (m.group(4), m.group(5)))
                r["healthy"] &= m.group(3) == "Healthy" and p.healthy
    finally:
        N.set_log_callback(None)
    out.append("sm_check=%d: median of 3 slices per suite (ms)" % ms)
    out.append("  %-20s %-22s %9s %9s %9s %9s  %s" % ("suite", "kernel per format", "kernel", "worker", "setup",
                                                     "call", "SMs / verdict"))
    for s in SUITES:
        r = rows[s]
        if not r["wall"]:
            out.append("  %-20s no slice" % s)
            continue
        kern = [statistics.median(k[f] for k in r["kernel"]) for f in range(3)]
        wall, call = statistics.median(r["wall"]), statistics.median(r["call"])
        out.append("  %-20s %-22s %9.1f %9.1f %9.1f %9.1f  %s %s" % (
            s, "/".join("%.1f" % x for x in kern), sum(kern), wall, wall - sum(kern), call, ",".join(sorted(r["sms"])),
            "Healthy" if r["healthy"] else "UNHEALTHY"))
    tot_wall = sum(statistics.median(rows[s]["wall"]) for s in SUITES if rows[s]["wall"])
    out.append("  one rotation: %.0f ms on the worker over 10 passes, %.1f ms per pass on average" % (tot_wall, tot_wall / 10))


def cli_runs(out):
    out.append("b200dp_cli <uri> cycle 40 [idle_ms], alternating (1 GiB ring, calib=3, min_frac=0.8)")
    for rep in range(2):
        for idle in (0, 1000):
            for uri in ("cuda:", "cuda:sm_check=10"):
                r = subprocess.run([CLI, uri, "cycle", "40", str(idle)], capture_output=True, text=True, timeout=600)
                line = r.stdout.strip().splitlines()[-1] if r.stdout.strip() else ""
                try:
                    j = json.loads(line)
                    out.append("  rep %d idle %4d %-18s exit %d wall_ms p50 %7.2f p99 %7.2f max %7.2f slowest_kernel_ms p50 "
                               "%.3f probe_frac_min %.4f" % (rep, idle, uri, r.returncode, j["wall_ms_median"],
                                                             j["wall_ms_p99"], j["wall_ms_max"],
                                                             j["slowest_kernel_ms_p50"], j["probe_frac_min"]))
                except (ValueError, KeyError):
                    out.append("  rep %d idle %4d %-18s exit %d: %s" % (rep, idle, uri, r.returncode,
                                                                       (r.stdout + r.stderr).strip()[-300:]))


def per_pass(pkg, out):
    N = pkg._native
    out.append("per pass, probe_health(timed=False): frac = in-kernel rate / calibrated ceiling; floor 0.8")
    for idle, n in ((0, 40), (1000, 10)):
        for uri in ("cuda:devices=0", "cuda:devices=0,sm_check=10"):
            with pkg.Context(uri) as ctx:
                fr, slow, after = [], 0, {}
                prev = 0
                for _ in range(n):
                    if idle:
                        time.sleep(idle / 1000.0)
                    (p,) = ctx.probe_health(timed=False)
                    fr.append(p.frac)
                    slow += bool(p.flags & N.RES_SLOW)
                    if prev:
                        after.setdefault(SUITES[prev - 1], []).append(p.frac)
                    prev = p.sm_check
                out.append("  idle %4d %-28s passes %d frac min %.4f median %.4f RES_SLOW %d" % (
                    idle, uri, n, min(fr), statistics.median(fr), slow))
                if after:
                    out.append("    frac min of the pass right after each suite's slice: " +
                               ", ".join("%s %.4f" % (s, min(v)) for s, v in after.items()))


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--out", default="", help="also write the report to this file")
    a = ap.parse_args()
    pkg = importlib.import_module("k8s-device-plugin_b200")
    out = ["card (name, power limit, max SM clock): " + card(), ""]
    # the CLI first: once this process holds a CUDA context, NVML lists it on the GPU, and the CLI's passes, seeing
    # another process there, rightly run no slice
    cli_runs(out)
    out.append("")
    for ms in (10, 100):
        slice_costs(pkg, ms, out)
        out.append("")
    per_pass(pkg, out)
    out.append("card at the end: " + card())
    text = "\n".join(out) + "\n"
    print(text)
    if a.out:
        os.makedirs(os.path.dirname(os.path.abspath(a.out)), exist_ok=True)
        with open(a.out, "w") as f:
            f.write(text)


if __name__ == "__main__":
    main()
