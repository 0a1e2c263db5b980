"""Anchored against unanchored nearest_pattern_in_each (DESIGN.md section 5.18) on the demultiplexing workload.

1 M DNA reads of 150 bases, each starting with one of 96 barcodes of 8-24 bases carrying 0-2 random edits
(substitution, insertion or deletion), the rest random bases; a resident DeviceSequenceSet.  Four arms, Levenshtein
and substitutions only, each unanchored and with anchor='start':
  * scan: the device time fzb_nearest_best_per_record reports (Haystack.nearest_best_per_record);
  * end to end: nearest_pattern_in_each on the resident set, host clock (the call ends in a device synchronise).
The arms alternate after a warm-up round; medians of --reps rounds.  The wrong-call rate is the share of reads whose
device answer is not the planted barcode; `tie` the share whose runner-up is at the winner's distance.

    python tools/probe_anchored.py [--reps 3] [--reads 1000000]

Prints the card, its power limit and max SM clock as nvidia-smi reports them; changes no setting."""
import argparse
import os
import statistics
import subprocess
import sys
import time

import numpy as np

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from fuzzysearch_b200 import DeviceSequenceSet, _native as F, nearest_pattern_in_each  # noqa: E402


def card():
    try:
        return subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                              capture_output=True, text=True, timeout=30).stdout.strip()
    except (OSError, subprocess.SubprocessError):
        return "unknown card"


def workload(rng, count):
    acgt = np.frombuffer(b"ACGT", dtype=np.uint8)
    codes = [bytes(acgt[rng.integers(0, 4, size=int(m))]) for m in rng.integers(8, 25, size=96)]
    truth = rng.integers(0, 96, size=count)
    tails = acgt[rng.integers(0, 4, size=(count, 160))]
    edits = rng.integers(0, 3, size=count)
    reads = []
    for i in range(count):
        b = bytearray(codes[truth[i]])
        for _ in range(int(edits[i])):
            kind, at, c = int(rng.integers(0, 3)), int(rng.integers(0, len(b))), int(acgt[rng.integers(0, 4)])
            if kind == 0:
                b[at] = c
            elif kind == 1:
                b.insert(at, c)
            elif len(b) > 1:
                del b[at]
        reads.append(bytes(b) + tails[i, :150 - len(b)].tobytes())
    return codes, truth, reads


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=3)
    ap.add_argument("--reads", type=int, default=1_000_000)
    a = ap.parse_args()
    rng = np.random.default_rng(7)
    codes, truth, reads = workload(rng, a.reads)
    seqset = DeviceSequenceSet(reads)
    print("card: %s" % card(), flush=True)
    arms = {(anchor, subs): None for subs in (False, True) for anchor in (None, "start")}

    def scan(anchor, subs):
        flags = (F.F_SUBSTITUTIONS_ONLY if subs else 0) | (F.F_ANCHOR_START if anchor else 0)
        with seqset._lock:
            pats = seqset._bind_many(codes)
            _, st = seqset._seq.haystack.nearest_best_per_record(pats, flags)
        return st

    def e2e(anchor, subs):
        t = time.perf_counter()
        rows = nearest_pattern_in_each(codes, seqset, substitutions_only=subs, anchor=anchor)
        return time.perf_counter() - t, rows

    for k in arms:  # warm-up
        scan(*k)
        e2e(*k)
    times = {k: ([], [], None, None) for k in arms}
    for _ in range(a.reps):
        for k in arms:
            st = scan(*k)
            dt, rows = e2e(*k)
            times[k][0].append(st["gpu_ms"])
            times[k][1].append(1e3 * dt)
            times[k] = (times[k][0], times[k][1], rows, st)
    for (anchor, subs), (scan_ms, e2e_ms, rows, st) in times.items():
        wrong = float(np.mean(rows.pattern != truth))
        tie = float(np.mean((rows.second_dist == rows.dist) & (rows.second_pattern >= 0)))
        print("%-13s %-12s scan %7.2f ms, end to end %7.2f ms, %6.2f G symbols read, wrong call %6.2f %%, "
              "second_dist == dist %6.2f %%  (route %s)"
              % ("substitutions" if subs else "levenshtein", "anchor=start" if anchor else "unanchored",
                 statistics.median(scan_ms), statistics.median(e2e_ms), st["bytes_scanned"] / 1e9, 100 * wrong,
                 100 * tie, st["route"]), flush=True)
    seqset.close()


if __name__ == "__main__":
    main()
