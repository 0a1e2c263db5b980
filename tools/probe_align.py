"""The alignments of matches on the device (align_in_each / fzb_align, DESIGN.md section 5.17) against what a user does
without them.

1. 1 M DNA reads of 150 bases x 96 barcodes of 20 bases: align_in_each over the best_match_in_each rows (max_l_dist=2)
   against the plain-Python restatement (tests/test_host_align.py) looped over the rows, timed on a sample and
   extrapolated.
2. The start recovery of nearest_pattern_in_each's rows on the same reads: align_in_each against find_nearest_matches
   per read (timed on a sample, extrapolated).
3. All matches of a Levenshtein search (m = 30, max_l_dist = 3) over a 4 GiB ACGT sequence with planted copies:
   fzb_align over the final list against the restatement on a sample.

Every arm's answers are compared on its sample.  The device arms report the median wall time of --reps calls after a
warm-up and the device time of the kernels (stats).

    python tools/probe_align.py [--reps 3] [--gib 4] [--reads 1000000]

Prints the card, its power limit and max SM clock as nvidia-smi reports them; changes no setting."""
import argparse
import os
import statistics
import subprocess
import sys
import time

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))
from fuzzysearch_b200 import (DeviceSequenceSet, _native as F, align_in_each, best_match_in_each,  # noqa: E402
                              find_nearest_matches, nearest_pattern_in_each)
from fuzzysearch_b200.search import _cigars  # noqa: E402
from test_host_align import BIG, align_anchored, cigar, free_start  # noqa: E402


def rand(rng, alphabet, n):
    a = np.frombuffer(alphabet, dtype=np.uint8)
    return a[rng.integers(0, len(a), size=n)]


def timed(f, reps):
    f()
    ts = []
    for _ in range(reps):
        t = time.perf_counter()
        out = f()
        ts.append(time.perf_counter() - t)
    return statistics.median(ts), out


def reads(rng, n, reps):
    bcs = [bytes(rand(rng, b"ACGT", 20)) for _ in range(96)]
    body = rand(rng, b"ACGT", n * 150).reshape(n, 150)
    for r in range(0, n, 2):
        b = bytearray(bcs[r % 96])
        b[int(rng.integers(0, 20))] = ord("A")
        if r % 6 == 0:
            del b[int(rng.integers(0, 19))]
        body[r, 10:10 + len(b)] = np.frombuffer(bytes(b), dtype=np.uint8)
    seqs = [bytes(x) for x in body]
    resident = DeviceSequenceSet(seqs)
    sample = rng.choice(n, size=1000, replace=False)

    best = best_match_in_each(bcs, resident, 2)
    t_dev, al = timed(lambda: align_in_each(bcs, resident, best, 2), reps)
    lim = (BIG, BIG, BIG, 2)
    t0 = time.perf_counter()
    want = {}
    for r in sample.tolist():
        if best.pattern[r] >= 0:
            s, e = int(best.start[r]), int(best.end[r])
            want[r] = cigar(align_anchored(bcs[best.pattern[r]], seqs[r][s:e], lim, int(best.dist[r]))[1])
    t_py = (time.perf_counter() - t0) / len(sample) * n
    assert all(al.cigar[r] == c for r, c in want.items())
    rows = int((best.pattern >= 0).sum())
    print("best_match_in_each rows: %d reads x %d barcodes, %d rows: align_in_each %.3f s, Python restatement %.1f s "
          "(extrapolated from %d reads); sample agrees" % (n, len(bcs), rows, t_dev, t_py, len(sample)), flush=True)

    near = nearest_pattern_in_each(bcs, resident)
    t_dev, al = timed(lambda: align_in_each(bcs, resident, near), reps)
    small = sample[:200].tolist()
    t0 = time.perf_counter()
    starts = {r: find_nearest_matches(bcs[near.pattern[r]], seqs[r]) for r in small}
    t_fnm = (time.perf_counter() - t0) / len(small) * n
    lev = (BIG, BIG, BIG, BIG)
    for r in small:
        s = free_start(bcs[near.pattern[r]], seqs[r], int(near.end[r]), 0, lev, int(near.dist[r]))
        assert al.start[r] == s and al.dist[r] == near.dist[r]
        # find_nearest_matches lists the consolidated matches at the same distance
        assert starts[r] and all(m.dist == near.dist[r] for m in starts[r])
    print("nearest_pattern_in_each start recovery: align_in_each %.3f s, find_nearest_matches per read %.1f s "
          "(extrapolated from %d reads); sample agrees" % (t_dev, t_fnm, len(small)), flush=True)
    resident.close()


def big_search(rng, gib, reps):
    n = gib << 30
    hs = F.Haystack.alloc(n)
    hs.fill_synthetic(b"ACGT", 3)
    P = bytes(rand(rng, b"ACGT", 30))
    for at in rng.integers(0, n - 64, size=100000).tolist():
        v = bytearray(P)
        v[int(rng.integers(0, 30))] = ord("C")
        if at % 3 == 0:
            del v[int(rng.integers(0, 29))]
        hs.write(at, bytes(v))
    res = hs.search_levenshtein(P, 3)
    s, e, d = res.arrays(F.FINAL)
    res.close()
    lev = (BIG, BIG, BIG, 3)

    def run():
        return hs.align([P], [BIG], [BIG], [BIG], [3], np.zeros(s.size), s, e, d)
    t_dev, (cols, ops, oo, st) = timed(run, reps)
    t_cig, cig = timed(lambda: _cigars(ops, oo, len(P) + cols[3], cols[1] >= 0), 1)
    idx = rng.choice(s.size, size=min(2000, s.size), replace=False).tolist()
    t0 = time.perf_counter()
    for i in idx:
        w = align_anchored(P, hs.read(int(s[i]), int(e[i] - s[i])), lev, int(d[i]))
        assert cig[i] == cigar(w[1])
    t_py = (time.perf_counter() - t0) / len(idx) * s.size
    print("%d GiB find_near_matches, m = 30, max_l_dist = 3: %d matches: fzb_align %.3f s (kernels %.2f ms), CIGARs "
          "%.3f s, Python restatement %.1f s (extrapolated from %d); sample agrees" %
          (gib, s.size, t_dev, st["gpu_ms"], t_cig, t_py, len(idx)), flush=True)
    hs.close()


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=3)
    ap.add_argument("--gib", type=int, default=4)
    ap.add_argument("--reads", type=int, default=1000000)
    args = ap.parse_args()
    print(subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv"],
                         capture_output=True, text=True).stdout.strip(), flush=True)
    rng = np.random.default_rng(1)
    reads(rng, args.reads, args.reps)
    big_search(rng, args.gib, args.reps)


if __name__ == "__main__":
    main()
