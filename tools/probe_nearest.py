"""find_nearest_matches / nearest_distance_in_each against the loop they replace -- find_near_matches with
max_l_dist = 0, 1, 2, ... until the list is non-empty -- on resident sequences (DESIGN.md section 5.14).

1. 4 GiB of synthetic ASCII and of ACGT, patterns of 20 / 32 / 64 symbols, one occurrence planted at distance 0, 2 or 5
   or none at all: the scan alone (time, rate, d*), then the whole find_nearest_matches (scan + search at d*) against
   the deepening loop on the same handle, and the equality of the two lists.  The deepening loop and the second stage
   are only run up to --max-dist (default 2; the searches at larger limits take the routes and meet the limits
   DESIGN.md section 8 describes); what is skipped is printed as not measured.
2. A million reads of 150 bases and a 25-base adapter: nearest_distance_in_each on a resident set against the same
   scan without records and against a per-read deepening loop, extrapolated from the first --loop-reads reads.

The arms alternate in one process after a warm-up round; medians of --reps rounds with their range.

    python tools/probe_nearest.py [--reps 3] [--gib 4] [--max-dist 2] [--loop-reads 10000]

Prints the card, its power limit and clocks as nvidia-smi reports them during the run; changes no setting."""
import argparse
import os
import statistics
import subprocess
import sys
import time

import numpy as np

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from fuzzysearch_b200 import (DeviceSequence, DeviceSequenceSet, _native as F, find_near_matches,  # noqa: E402
                              find_nearest_matches, nearest_distance_in_each)

ASCII = bytes(range(32, 127))


def spread(xs):
    return "%.2f (%.2f-%.2f)" % (statistics.median(xs), min(xs), max(xs))


def mutate(rng, pat, alphabet, d):
    """d substitutions at distinct places, each to another letter"""
    v = bytearray(pat)
    for i in rng.choice(len(v), size=d, replace=False).tolist():
        v[i] = next(c for c in alphabet if c != v[i])
    return bytes(v)


def deepen(pat, seq):
    """-> the first non-empty list, or None when a guess runs into a limit of its route (DESIGN.md section 8)"""
    k = 0
    while True:
        try:
            found = find_near_matches(pat, seq, max_l_dist=k)
        except F.UnsupportedError:
            return None
        if found:
            return found
        k += 1


def whole_sequences(rng, n, reps, max_dist):
    for name, alphabet in (("ASCII", ASCII), ("ACGT", b"ACGT")):
        hs = F.Haystack.alloc(n)
        hs.fill_synthetic(alphabet, 7)
        seq = DeviceSequence(_haystack=hs)
        for m in (20, 32, 64):
            pat = bytes(rng.choice(np.frombuffer(alphabet, np.uint8), size=m))
            for planted in (0, 2, 5, None):
                at = n // 3 * 2 + 12345
                saved = hs.read(at, m)
                if planted is not None:
                    hs.write(at, mutate(rng, pat, alphabet, planted))
                scans, nearest_ms, loop_ms = [], [], []
                compare = planted is not None and planted <= max_dist
                for rep in range(reps + 1):  # (the first round warms both arms up)
                    d, n_ends, first, st = hs.nearest_distance(pat)
                    if rep:
                        scans.append(st["gpu_ms"])
                    if compare:
                        t0 = time.perf_counter()
                        a = find_nearest_matches(pat, seq)
                        t1 = time.perf_counter()
                        b = deepen(pat, seq)
                        t2 = time.perf_counter()
                        assert a == b, (name, m, planted, a, b)
                        if rep:
                            nearest_ms.append((t1 - t0) * 1e3)
                            loop_ms.append((t2 - t1) * 1e3)
                ms = statistics.median(scans)
                print("%s %.2f GiB, m=%d, planted at %s: d*=%d n_ends=%d | scan ms %s, %.0f GB/s | %s" % (
                    name, n / 2.0 ** 30, m, planted, d, n_ends, spread(scans), n / ms / 1e6,
                    "find_nearest_matches ms %s, deepening loop ms %s, lists equal" % (spread(nearest_ms), spread(loop_ms))
                    if compare else "second stage and deepening loop not measured"), flush=True)
                hs.write(at, saved)
        hs.close()


def reads(rng, count, reps, loop_reads):
    adapter = b"AGATCGGAAGAGCACACGTCTGAAC"
    rows = np.frombuffer(b"ACGT", np.uint8)[rng.integers(0, 4, size=(count, 150))]
    for r in range(0, count, 3):
        p = int(rng.integers(0, 125))
        rows[r, p:p + 25] = np.frombuffer(mutate(rng, adapter, b"ACGT", int(rng.integers(0, 4))), np.uint8)
    seqs = [r.tobytes() for r in rows]
    resident = DeviceSequenceSet(seqs)
    flat = DeviceSequence(b"\0".join(seqs) + b"\0")
    timed = {"in_each": [], "scan per record": [], "scan without records": []}
    for rep in range(reps + 1):
        t0 = time.perf_counter()
        got = nearest_distance_in_each(adapter, resident)
        t1 = time.perf_counter()
        with resident._lock:
            st_rec = resident._seq.haystack.nearest_per_record(resident._bind(adapter))[2]
        st_flat = flat.haystack.nearest_distance(adapter)[3]
        if rep:
            for key, v in zip(timed, ((t1 - t0) * 1e3, st_rec["gpu_ms"], st_flat["gpu_ms"])):
                timed[key].append(v)
    t0 = time.perf_counter()
    refused = 0
    for r in range(loop_reads):
        found = deepen(adapter, seqs[r])
        refused += found is None
        assert found is None or found[0].dist == got.dist[r]
    loop_s = time.perf_counter() - t0
    print("%d reads of 150 bases, adapter of 25: nearest_distance_in_each end to end ms %s | scan ms: per record %s, "
          "without records %s | per-read deepening loop %.1f s for %d reads (%d of them ended in a refusal) = %.0f s for all "
          "(extrapolated)" % (
              count, spread(timed["in_each"]), spread(timed["scan per record"]), spread(timed["scan without records"]),
              loop_s, loop_reads, refused, loop_s * count / loop_reads), flush=True)
    resident.close()
    flat.close()


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=3)
    ap.add_argument("--gib", type=float, default=4.0)
    ap.add_argument("--max-dist", type=int, default=2)
    ap.add_argument("--reads", type=int, default=1_000_000)
    ap.add_argument("--loop-reads", type=int, default=10_000)
    args = ap.parse_args()
    print(subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.sm,clocks.max.sm,clocks.mem",
                          "--format=csv"], capture_output=True, text=True).stdout.strip(), flush=True)
    rng = np.random.default_rng(5)
    reads(rng, args.reads, args.reps, min(args.loop_reads, args.reads))
    whole_sequences(rng, int(args.gib * 2 ** 30) // 128 * 128, args.reps, args.max_dist)


if __name__ == "__main__":
    main()
