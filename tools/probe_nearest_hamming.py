"""The nearest calls under substitutions only (DESIGN.md section 5.16) against what a user does without them, on
resident inputs.

1. One pattern over 4 GiB of ASCII and of ACGT, m = 20 / 32 / 64: the substitutions-only scan's device time next to
   the Levenshtein scan's on the same data; find_nearest_matches(substitutions_only=True) against the deepening loop
   of substitutions-only find_near_matches (k = 0, 1, ... until a list comes back), with an occurrence planted at 0
   and at 2 substitutions (m = 20).
2. 1 M DNA reads of 150 bases x 96 barcodes of 8-24 bases: nearest_pattern_in_each(substitutions_only=True) against
   best_match_in_each(max_substitutions=2, max_insertions=0, max_deletions=0) and against a loop of
   nearest_distance_in_each(substitutions_only=True) plus the numpy reduction.
3. 1 M reads x one 25-base adapter: nearest_distance_in_each(substitutions_only=True).

The arms alternate after a warm-up round; medians of --reps rounds.  Every arm's answers are compared with the
others'.  Scan rates are the bytes scanned over the device time the call reports.

    python tools/probe_nearest_hamming.py [--reps 3] [--gib 4] [--reads 1000000]

Prints the card, its power limit and max SM clock as nvidia-smi reports them; changes no setting."""
import argparse
import os
import statistics
import subprocess
import sys
import time

import numpy as np

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from fuzzysearch_b200 import (DeviceSequence, DeviceSequenceSet, _native as F, best_match_in_each,  # noqa: E402
                              find_near_matches, find_nearest_matches, nearest_distance_in_each,
                              nearest_pattern_in_each)

SUB = F.F_SUBSTITUTIONS_ONLY


def med(xs):
    return statistics.median(xs)


def rand(rng, alphabet, n):
    a = np.frombuffer(alphabet, dtype=np.uint8)
    return a[rng.integers(0, len(a), size=n, dtype=np.uint8)]


def rounds(arms, reps):
    """-> per arm: (median seconds, median of the arm's second value, last answer); a warm-up round first"""
    for f in arms.values():
        f()
    got = {k: [] for k in arms}
    for _ in range(reps):
        for k, f in arms.items():
            t = time.perf_counter()
            extra, answer = f()
            got[k].append((time.perf_counter() - t, extra, answer))
    return {k: (med([x[0] for x in v]), med([x[1] for x in v]), v[-1][2]) for k, v in got.items()}


def one_pattern(rng, n, reps):
    block = 1 << 28
    for name, alphabet in (("ASCII", bytes(range(32, 127))), ("ACGT", b"ACGT")):
        S = np.tile(rand(rng, alphabet, block), n // block)
        pats = {m: bytes(rand(rng, alphabet, m)) for m in (20, 32, 64)}
        hs = F.Haystack.from_host(S)
        for m, P in pats.items():
            def scan(flags):
                got = hs.nearest_distance(P, flags)
                return got[3]["gpu_ms"], got[:3]

            r = rounds({"hamming": lambda: scan(SUB), "levenshtein": lambda: scan(0)}, reps)
            d, n_ends, first = r["hamming"][2]
            print("%s %d bytes, m = %d: substitutions-only scan %.2f ms (%.2f TB/s), Levenshtein scan %.2f ms "
                  "(%.2f TB/s); d* = %d, %d ends, first at %d"
                  % (name, S.size, m, r["hamming"][1], S.size / r["hamming"][1] / 1e9, r["levenshtein"][1],
                     S.size / r["levenshtein"][1] / 1e9, d, n_ends, first), flush=True)
        hs.close()
        P = pats[20]
        for subs in (0, 2):
            v = np.frombuffer(P, dtype=np.uint8).copy()
            v[[3, 11][:subs]] = ord("~") if name == "ASCII" else ord("N")
            at = S.size // 3 + 12345
            S[at:at + 20] = v
            ds = DeviceSequence(S)

            def nearest():
                ms = find_nearest_matches(P, ds, substitutions_only=True)
                return 0.0, [(x.start, x.end, x.dist) for x in ms]

            def deepening():
                k = 0
                while True:
                    ms = find_near_matches(P, ds, max_substitutions=k, max_insertions=0, max_deletions=0)
                    if ms:
                        return float(k), [(x.start, x.end, x.dist) for x in ms]
                    k += 1

            r = rounds({"nearest": nearest, "deepening": deepening}, reps)
            assert r["nearest"][2] == r["deepening"][2], (name, subs)
            print("%s, m = 20, occurrence at %d substitutions: find_nearest_matches %.1f ms, deepening loop %.1f ms "
                  "(to k = %d); %d matches, equal lists" % (name, subs, 1e3 * r["nearest"][0],
                                                            1e3 * r["deepening"][0], r["deepening"][1],
                                                            len(r["nearest"][2])), flush=True)
            ds.close()
            S[at:at + 20] = rand(rng, alphabet, 20)
        del S


def fold(columns, i, dist, end):
    """pattern i's (dist, end) of every record folded into the five columns; -1 (no window) is left out"""
    pattern, best, at, pat2, dist2 = columns
    has = dist >= 0
    first = has & ((pattern < 0) | (dist < best))
    second = has & ~first & ((pat2 < 0) | (dist < dist2))
    pat2[first], dist2[first] = pattern[first], best[first]
    pattern[first], best[first], at[first] = i, dist[first], end[first]
    pat2[second], dist2[second] = i, dist[second]


def reads_barcodes(rng, count, reps):
    rows = rand(rng, b"ACGT", count * 150).reshape(count, 150).copy()
    barcodes = [bytes(rand(rng, b"ACGT", int(m))) for m in rng.integers(8, 25, size=96)]
    for r in range(0, count, 2):
        b = np.frombuffer(barcodes[r % 96], dtype=np.uint8).copy()
        b[rng.integers(0, len(b), size=int(rng.integers(0, 4)))] = ord("N")
        rows[r, 10:10 + len(b)] = b
    seqset = DeviceSequenceSet([r.tobytes() for r in rows])
    hay = seqset._seq.haystack
    bound = seqset._bind_many(barcodes)

    def nearest():
        got = nearest_pattern_in_each(barcodes, seqset, substitutions_only=True)
        return 0.0, (got.pattern, got.dist, got.end, got.second_pattern, got.second_dist)

    def best():
        got = best_match_in_each(barcodes, seqset, max_substitutions=2, max_insertions=0, max_deletions=0)
        return 0.0, (got.pattern, got.dist, got.end, got.second_pattern, got.second_dist)

    def loop():
        cols = tuple(np.full(count, -1, dtype=ty) for ty in (np.int32, np.int32, np.int64, np.int32, np.int32))
        for i, p in enumerate(bound):
            d, e, _ = hay.nearest_per_record(p, SUB)
            fold(cols, i, d, e)
        return 0.0, cols

    r = rounds({"nearest": nearest, "best_match": best, "loop": loop}, reps)
    a, b, c = r["nearest"][2], r["best_match"][2], r["loop"][2]
    assert all(np.array_equal(x, y) for x, y in zip(a, c))
    near = a[1] <= 2
    assert np.array_equal(b[0] >= 0, near) and all(np.array_equal(x[near], y[near]) for x, y in zip(a[:3], b[:3]))
    scan = hay.nearest_best_per_record(bound, SUB)[1]["gpu_ms"]
    print("%d reads x 96 barcodes: nearest_pattern_in_each %.1f ms (scans %.2f ms), best_match_in_each "
          "(2 substitutions) %.1f ms, loop + reduction %.1f ms; equal rows (best_match where dist <= 2)"
          % (count, 1e3 * r["nearest"][0], scan, 1e3 * r["best_match"][0], 1e3 * r["loop"][0]), flush=True)
    adapter = b"AGATCGGAAGAGCACACGTCTGAAC"
    for r_ in range(1, count, 3):
        rows[r_, 60:85] = np.frombuffer(adapter, dtype=np.uint8)
    seqset.close()
    seqset = DeviceSequenceSet([r.tobytes() for r in rows])

    def adapter_arm():
        got = nearest_distance_in_each(adapter, seqset, substitutions_only=True)
        return 0.0, (got.dist, got.end)

    r = rounds({"adapter": adapter_arm}, reps)
    H = np.zeros((1000, 126), dtype=np.int16)
    for j in range(25):
        H += rows[:1000, j:j + 126] != adapter[j]
    d, e = r["adapter"][2]
    assert np.array_equal(d[:1000], H.min(axis=1)) and np.array_equal(e[:1000], H.argmin(axis=1) + 25)
    scan = seqset._seq.haystack.nearest_per_record(seqset._bind(adapter), SUB)[2]["gpu_ms"]
    print("%d reads x one 25-base adapter: nearest_distance_in_each %.1f ms (scan %.2f ms)"
          % (count, 1e3 * r["adapter"][0], scan), flush=True)
    seqset.close()


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=3)
    ap.add_argument("--gib", type=int, default=4)
    ap.add_argument("--reads", type=int, default=1_000_000)
    args = ap.parse_args()
    print(subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv"],
                         capture_output=True, text=True).stdout.strip(), flush=True)
    rng = np.random.default_rng(1)
    reads_barcodes(rng, args.reads, args.reps)
    one_pattern(rng, args.gib << 30, args.reps)


if __name__ == "__main__":
    main()
