"""nearest_pattern_in_each / nearest_distance_batch against the loops they replace, on resident inputs (DESIGN.md
section 5.15).

1. 1 M DNA reads of 150 bases x 96 barcodes of 8-24 bases: nearest_pattern_in_each against a loop of
   nearest_distance_in_each (its per-record call on the resident handle) plus the numpy reduction.
2. 2 M ASCII lines of 40-120 bytes x 1 024 terms of 6-32 bytes: the same two arms.
3. 4 GiB of ASCII and of ACGT x 64 patterns of 20 / 32 / 64 symbols: nearest_distance_batch against a loop of
   nearest_distance.

For each: end-to-end time, device time of the scans (the calls' stats), and issue slots per byte*pattern,
3.3e13 * t / (N * P), where 3.3e13 = 132 SMs x 4 schedulers x 1.98 GHz x 32 lanes (the measure DESIGN.md section 5.14
gives the single-pattern scan).  The loops reduce on the host pattern by pattern, as nearest_pattern_in_each's
fallback does.  The arms alternate after a warm-up round; medians of --reps rounds.  The answers of both arms are
compared.

    python tools/probe_nearest_batch.py [--reps 3] [--gib 4]

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

SLOTS = 3.3e13


def med(xs):
    return statistics.median(xs)


def rand(rng, alphabet, n):
    a = np.frombuffer(alphabet, dtype=np.uint8)
    return a[rng.integers(0, len(a), size=n, dtype=np.uint8 if len(a) < 256 else np.int64)]


def fold(columns, i, dist, end):
    """pattern i's (dist, end) of every record folded into the five columns (ties: the smaller index stays)"""
    pattern, best, at, pat2, dist2 = columns
    first = (pattern < 0) | (dist < best)
    second = ~first & ((pat2 < 0) | (dist < dist2))
    pat2[first], dist2[first] = pattern[first], best[first]
    pattern[first], best[first], at[first] = i, dist[first], end[first]
    pat2[second], dist2[second] = i, dist[second]


def record_workload(name, rng, reads, pats, reps):
    seqset = DeviceSequenceSet(reads)
    hay = seqset._seq.haystack
    n_bytes = int(seqset.offsets[-1])
    bound = seqset._bind_many(pats)

    def batch():  # end to end through the public call; the device time from the same call on the handle
        t = time.perf_counter()
        got = nearest_pattern_in_each(pats, seqset)
        t = time.perf_counter() - t
        return t, hay.nearest_best_per_record(bound)[1]["gpu_ms"], (got.pattern, got.dist, got.end,
                                                                    got.second_pattern, got.second_dist)

    def loop():
        t, dev = time.perf_counter(), 0.0
        cols = tuple(np.full(len(reads), -1, dtype=ty) for ty in (np.int32, np.int32, np.int64, np.int32, np.int32))
        for i, p in enumerate(bound):
            d, e, st = hay.nearest_per_record(p)
            dev += st["gpu_ms"]
            fold(cols, i, d, e)
        return time.perf_counter() - t, dev, cols

    batch(), loop()
    tb, tl, kb, kl = [], [], [], []
    for _ in range(reps):
        a, ka, ca = batch()
        b, kb_, cb = loop()
        tb.append(a), kb.append(ka), tl.append(b), kl.append(kb_)
    same = all(np.array_equal(x, y) for x, y in zip(ca, cb))
    assert same, name
    kbm = med(kb) / 1e3
    print("%s: nearest_pattern_in_each %.1f ms end to end (scans %.2f ms; %.1f slots per byte*pattern), "
          "loop %.1f ms (scans %.2f ms; %.1f slots per byte*pattern); equal rows: %s"
          % (name, 1e3 * med(tb), med(kb), SLOTS * kbm / (n_bytes * len(pats)), 1e3 * med(tl), med(kl),
             SLOTS * med(kl) / 1e3 / (n_bytes * len(pats)), same), flush=True)
    seqset.close()


def whole_workload(name, rng, n, alphabet, reps):
    S = rand(rng, alphabet, n)
    pats = [bytes(rand(rng, alphabet, m)) for m in [20] * 22 + [32] * 21 + [64] * 21]
    hs = F.Haystack.from_host(S)

    def batch():
        t = time.perf_counter()
        d, e, st = hs.nearest_distance_batch(pats)
        return time.perf_counter() - t, st["gpu_ms"], (d.tolist(), e.tolist())

    def loop():
        t, dev, d, e = time.perf_counter(), 0.0, [], []
        for p in pats:
            x, _, f, st = hs.nearest_distance(p)
            dev += st["gpu_ms"]
            d.append(x)
            e.append(f)
        return time.perf_counter() - t, dev, (d, e)

    batch(), loop()
    tb, tl, kb, kl = [], [], [], []
    for _ in range(reps):
        a, ka, ra = batch()
        b, kb_, rb = loop()
        tb.append(a), kb.append(ka), tl.append(b), kl.append(kb_)
    assert ra == rb, name
    print("%s 4 GiB-class (%d bytes) x 64 patterns: nearest_distance_batch %.1f ms end to end (scans %.2f ms; "
          "%.1f slots per byte*pattern), nearest_distance loop %.1f ms (scans %.2f ms; %.1f); equal: True"
          % (name, n, 1e3 * med(tb), med(kb), SLOTS * med(kb) / 1e3 / (n * 64), 1e3 * med(tl), med(kl),
             SLOTS * med(kl) / 1e3 / (n * 64)), flush=True)
    hs.close()
    del S


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=3)
    ap.add_argument("--gib", type=float, default=4)
    ap.add_argument("--reads", type=int, default=1_000_000)
    ap.add_argument("--lines", type=int, default=2_000_000)
    args = ap.parse_args()
    print(subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv"],
                         capture_output=True, text=True).stdout.strip(), flush=True)
    rng = np.random.default_rng(1)
    rows = rand(rng, b"ACGT", args.reads * 150).reshape(args.reads, 150)
    barcodes = [bytes(rand(rng, b"ACGT", int(m))) for m in rng.integers(8, 25, size=96)]
    reads = [r.tobytes() for r in rows]
    record_workload("1 M reads x 96 barcodes", rng, reads, barcodes, args.reps)
    del reads, rows
    ascii_ = bytes(range(32, 127))
    text = rand(rng, ascii_, args.lines * 120).tobytes()
    lens = rng.integers(40, 121, size=args.lines)
    lines, at = [], 0
    for n in lens.tolist():
        lines.append(text[at:at + n])
        at += n
    terms = [bytes(rand(rng, ascii_, int(m))) for m in rng.integers(6, 33, size=1024)]
    record_workload("2 M lines x 1 024 terms", rng, lines, terms, args.reps)
    del lines, text
    n = int(args.gib * (1 << 30))
    for name, alphabet in (("ASCII", ascii_), ("ACGT", b"ACGT")):
        whole_workload(name, rng, n, alphabet, args.reps)


if __name__ == "__main__":
    main()
