"""best_match_in_each against find_near_matches_batch_in_each followed by the same reduction in Python, on resident
sets (DESIGN.md section 5.13).  Three workloads: 96 DNA barcodes (1..2 substitutions) over a million reads, the same
barcodes with max_l_dist = 1, and 1 024 ASCII terms of mixed classes over two million lines.  The arms alternate; every
row of the first 10 000 records is compared.  Per workload: end-to-end medians with ranges, the handle's stream time
around fzb_best_per_record (fzb_timer: kernels, copies and the gaps between passes), the passes' own kernel time from
its stats (which leaves the reducing kernels out), and the stream time around the batch arm's searches.

    python tools/probe_best_match.py [--reps 3] [--scale 1.0]

Prints the card, its power limit and clocks as nvidia-smi reports them during the run; changes no setting."""
import argparse
import os
import statistics
import subprocess
import sys
import time

import numpy as np

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from fuzzysearch_b200 import DeviceSequenceSet, best_match_in_each, find_near_matches_batch_in_each  # noqa: E402

DNA, ASCII = np.frombuffer(b"ACGT", np.uint8), np.arange(32, 127, dtype=np.uint8)
NAMES = ("pattern", "start", "end", "dist", "second_pattern", "second_dist")


def substitute(rng, pat, alpha):
    v = bytearray(pat)
    v[int(rng.integers(len(v)))] = int(alpha[int(rng.integers(len(alpha)))])
    return bytes(v)


def reads_and_barcodes(rng, n):
    reads = DNA[rng.integers(0, 4, size=(n, 150))]
    codes = [bytes(DNA[rng.integers(0, 4, size=int(m))]) for m in rng.integers(8, 25, size=96)]
    for i in range(0, n, 3):
        v = np.frombuffer(substitute(rng, codes[int(rng.integers(96))], DNA), np.uint8)
        p = int(rng.integers(0, 150 - len(v) + 1))
        reads[i, p:p + len(v)] = v
    return [r.tobytes() for r in reads], codes


def lines_and_terms(rng, n):
    lengths = rng.integers(20, 120, size=n)
    flat = ASCII[rng.integers(0, len(ASCII), size=int(lengths.sum()))]
    ends = np.cumsum(lengths)
    terms, lim = [], dict(max_substitutions=[], max_insertions=[], max_deletions=[], max_l_dist=[])
    for q in range(1024):
        m = int(rng.integers(6, 33))
        terms.append(bytes(ASCII[rng.integers(0, len(ASCII), size=m)]))
        k = 0 if q % 4 == 0 else 1 if m < 16 else 2
        for name, v in zip(lim, [(0, 0, 0), (k, 0, 0), (k, k, k), (k, 1, 0)][q % 4] + (k,)):
            lim[name].append(v)
    for r in rng.choice(n, size=n // 4, replace=False).tolist():
        v = substitute(rng, terms[int(rng.integers(1024))], ASCII)
        if lengths[r] >= len(v):
            p = int(ends[r] - lengths[r] + rng.integers(0, lengths[r] - len(v) + 1))
            flat[p:p + len(v)] = np.frombuffer(v, np.uint8)
    blob = flat.tobytes()
    return [blob[e - l:e] for e, l in zip(ends.tolist(), lengths.tolist())], terms, lim


def reduce_dicts(dicts, n):
    """the rows of best_match_in_each from find_near_matches_batch_in_each's dicts"""
    cols = [np.full(n, -1, dtype=np.int64) for _ in NAMES]
    pat, start, end, dist, pat2, dist2 = cols
    for i, d in enumerate(dicts):
        for r, ms in d.items():
            m = min(ms, key=lambda x: (x.dist, x.start - x.end, x.start))
            if pat[r] < 0 or m.dist < dist[r]:
                pat2[r], dist2[r] = pat[r], dist[r]
                pat[r], start[r], end[r], dist[r] = i, m.start, m.end, m.dist
            elif pat2[r] < 0 or m.dist < dist2[r]:
                pat2[r], dist2[r] = i, m.dist
    return cols


def spread(xs):
    return "%.1f (%.1f-%.1f)" % (statistics.median(xs), min(xs), max(xs))


def run(name, pats, seqs, lim, reps):
    resident = DeviceSequenceSet(seqs)
    hs = resident._seq.haystack
    timed = {"best": [], "best stream": [], "batch+reduce": [], "batch stream": []}
    matches = 0
    for rep in range(reps + 1):  # (the first round warms both arms up)
        hs.timer_start()
        t0 = time.perf_counter()
        best = best_match_in_each(pats, resident, **lim)
        t1 = time.perf_counter()
        stream_best = hs.timer_stop()
        hs.timer_start()
        t2 = time.perf_counter()
        dicts = find_near_matches_batch_in_each(pats, resident, **lim)
        stream_batch = hs.timer_stop()
        cols = reduce_dicts(dicts, len(seqs))
        t3 = time.perf_counter()
        matches = sum(len(ms) for d in dicts for ms in d.values())
        for name_, col in zip(NAMES, cols):
            assert np.array_equal(getattr(best, name_)[:10000], col[:10000]), (name, name_)
        if rep:
            for key, v in zip(timed, ((t1 - t0) * 1e3, stream_best, (t3 - t2) * 1e3, stream_batch)):
                timed[key].append(v)
    from fuzzysearch_b200.common import LevenshteinSearchParams
    params = [LevenshteinSearchParams(*[v[q] if isinstance(v, list) else v for v in (
        lim.get("max_substitutions"), lim.get("max_insertions"), lim.get("max_deletions"), lim.get("max_l_dist"))])
        for q in range(len(pats))]
    with resident._lock:
        _, stats = hs.best_per_record(resident._bind_many(pats), *zip(*[p.unpacked for p in params]))
    print("%s: %d patterns x %d records, %d matches in the lists | end to end ms: best_match_in_each %s, batch + Python "
          "reduction %s | stream ms: best %s, batch %s | passes' kernel ms %.1f, launches %d" % (
              name, len(pats), len(seqs), matches, spread(timed["best"]), spread(timed["batch+reduce"]),
              spread(timed["best stream"]), spread(timed["batch stream"]), stats["gpu_ms"], stats["n_launches"]),
          flush=True)
    resident.close()


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=3)
    ap.add_argument("--scale", type=float, default=1.0)
    args = ap.parse_args()
    print(subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.sm,clocks.max.sm,clocks.mem",
                          "--format=csv"], capture_output=True, text=True).stdout.strip(), flush=True)
    rng = np.random.default_rng(5)
    reads, codes = reads_and_barcodes(rng, int((1 << 20) * args.scale))
    run("barcodes, 1..2 substitutions", codes, reads,
        dict(max_substitutions=[1 + q % 2 for q in range(96)], max_insertions=0, max_deletions=0), args.reps)
    run("barcodes, max_l_dist 1", codes, reads, dict(max_l_dist=1), args.reps)
    del reads
    lines, terms, lim = lines_and_terms(rng, int(2_000_000 * args.scale))
    run("ASCII terms, mixed classes", terms, lines, lim, args.reps)


if __name__ == "__main__":
    main()
