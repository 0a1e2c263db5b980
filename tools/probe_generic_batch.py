"""Generic-limit batch (fzb_search_generic_batch) against one search per pattern, on a haystack generated on the
device: for each workload the warmed batch time (device stopwatch around the call and the read-back of every list),
the shared scans' kernel time, their candidates, the patterns per route, the summed one-by-one search_generic time of
the same patterns on the same handle, and whether every list equals its single search.  Prints one JSON line with
the card's name and power limit.

    python tools/probe_generic_batch.py [--n BYTES] [--patterns 1024] [--workloads ascii,dna]
"""
import argparse
import json
import os
import sys
from collections import Counter

sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import numpy as np

from fuzzysearch_b200 import _native as F
from probe_ham_batch import card, lists, same

SHARED = ("generic-ngrams/batch-scan", "generic-lp/batch-scan")
# name -> (alphabet, pattern lengths)
WORKLOADS = {"ascii": (bytes(range(32, 127)), (12, 64)), "dna": (b"ACGT", (12, 64))}


def draw_limits(rng):
    """normalised generic limits (subs, ins, dels, max_l): subs 0-3, ins 0-1, dels 0-1, at least one insertion or
    deletion, and a total above the smallest per-operation limit (else the search class is not GenericSearch)"""
    subs, ins, dels = int(rng.integers(0, 4)), int(rng.integers(0, 2)), int(rng.integers(0, 2))
    if ins == 0 and dels == 0:
        ins = 1
    lo, hi = min(subs, ins, dels) + 1, subs + ins + dels
    l = int(rng.integers(lo, hi + 1))
    return min(subs, l), min(ins, l), min(dels, l), l


def workload(name, n, count=1024, plants=8, seed=20261015):
    """-> (alphabet, patterns, limits, writes): `count` random patterns, each planted `plants` times in [0, n) with
    at most max_subs substitutions and, if allowed, one deletion; writes = [(position, bytes)]."""
    alphabet, (mlo, mhi) = WORKLOADS[name]
    rng = np.random.default_rng(seed)
    alpha = np.frombuffer(alphabet, dtype=np.uint8)
    pats, limits, writes = [], [], []
    for _ in range(count):
        m = int(rng.integers(mlo, mhi + 1))
        lim = draw_limits(rng)
        p = alpha[rng.integers(0, len(alpha), size=m)]
        pats.append(p.tobytes())
        limits.append(lim)
        for _ in range(plants):
            v = p.copy()
            idx = rng.choice(m, size=int(rng.integers(0, lim[0] + 1)), replace=False)
            v[idx] = alpha[rng.integers(0, len(alpha), size=idx.size)]
            if lim[2] and lim[0] < lim[3] and rng.integers(0, 2):
                v = np.delete(v, int(rng.integers(0, m)))
            writes.append((int(rng.integers(0, n - m)), v.tobytes()))
    return alphabet, pats, limits, writes


def make_haystack(name, n, count=1024, seed=20261015):
    """-> (handle holding the workload's synthetic sequence with its plants, patterns, limits)"""
    alphabet, pats, limits, writes = workload(name, n, count, seed=seed)
    hs = F.Haystack.alloc(n)
    hs.fill_synthetic(alphabet, seed)
    for pos, v in writes:
        hs.write(pos, v)
    return hs, pats, limits


def batch(hs, pats, limits, flags=0):
    return hs.search_generic_batch(pats, *zip(*limits), flags=flags) if pats else ([], {})


def measure(hs, pats, limits):
    warm, _ = batch(hs, pats[:64], limits[:64])  # warm-up: module load, pass buffers, byte statistics
    for r in warm:
        r.close()
    hs.timer_start()
    results, _ = batch(hs, pats, limits)
    got = [lists(r) for r in results]
    batch_ms = hs.timer_stop()
    stats = [r.stats() for r in results]
    for r in results:
        r.close()
    shared = [s for s in stats if s["route"] in SHARED]
    one = hs.search_generic(pats[0], *limits[0])  # warm-up of the single search
    one.close()
    single_ms, equal = 0.0, True
    for p, lim, g in zip(pats, limits, got):
        hs.timer_start()
        one = hs.search_generic(p, *lim)
        want = lists(one)
        single_ms += hs.timer_stop()
        one.close()
        equal &= same(g, want)
    return {"batch_ms": round(batch_ms, 3),
            "scan_ms": round(sum(s["gpu_ms"] for s in shared if s["bytes_scanned"]), 3),
            "passes": sum(1 for s in shared if s["bytes_scanned"]),
            "candidates": int(sum(s["n_candidates"] for s in shared)),
            "routes": dict(Counter(s["route"] for s in stats)),
            "one_by_one_ms": round(single_ms, 3),
            "matches": int(sum(len(g[0][0]) for g in got)),
            "all_equal_single": bool(equal)}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--n", type=int, default=4 << 30)
    ap.add_argument("--patterns", type=int, default=1024)
    ap.add_argument("--workloads", default="ascii,dna")
    a = ap.parse_args()
    if F.device_count() == 0:
        raise SystemExit("no CUDA device")
    name, power = card()
    out = {"card": name, "power_limit": power, "n": a.n, "patterns": a.patterns}
    for w in a.workloads.split(","):
        hs, pats, limits = make_haystack(w, a.n, a.patterns)
        out[w] = measure(hs, pats, limits)
        hs.close()
    print(json.dumps(out))


if __name__ == "__main__":
    main()
