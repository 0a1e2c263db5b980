"""Substitutions-only batch (fzb_search_hamming_batch) against one search per pattern, on a haystack generated on the
device: for each workload the warmed batch time (device stopwatch around the call and the read-back of every list),
the shared scans' kernel time, their candidates, the patterns per route, the summed one-by-one search_hamming time of
the same patterns on the same handle, and whether every list equals its single search.  Prints one JSON line with
the card's name and power limit.

    python tools/probe_ham_batch.py [--n BYTES] [--patterns 1024] [--workloads dna,ascii]
"""
import argparse
import json
import os
import subprocess
import sys
from collections import Counter

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import numpy as np

from fuzzysearch_b200 import _native as F

SHARED = "hamming/batch-scan"
# name -> (alphabet, pattern lengths, substitution budgets)
WORKLOADS = {"dna": (b"ACGT", (20, 32), (1, 3)), "ascii": (bytes(range(32, 127)), (12, 64), (1, 4))}


def workload(name, n, count=1024, plants=8, seed=20261015):
    """-> (alphabet, patterns, ks, writes): `count` random patterns, each planted `plants` times in [0, n) with at
    most k substitutions; writes = [(position, bytes)]."""
    alphabet, (mlo, mhi), (klo, khi) = WORKLOADS[name]
    rng = np.random.default_rng(seed)
    alpha = np.frombuffer(alphabet, dtype=np.uint8)
    pats, ks, writes = [], [], []
    for _ in range(count):
        m, k = int(rng.integers(mlo, mhi + 1)), int(rng.integers(klo, khi + 1))
        p = alpha[rng.integers(0, len(alpha), size=m)]
        pats.append(p.tobytes())
        ks.append(k)
        for _ in range(plants):
            v = p.copy()
            idx = rng.choice(m, size=int(rng.integers(0, k + 1)), replace=False)
            v[idx] = alpha[rng.integers(0, len(alpha), size=idx.size)]
            writes.append((int(rng.integers(0, n - m)), v.tobytes()))
    return alphabet, pats, ks, writes


def make_haystack(name, n, count=1024, seed=20261015):
    """-> (handle holding the workload's synthetic sequence with its plants, patterns, ks)"""
    alphabet, pats, ks, writes = workload(name, n, count, seed=seed)
    hs = F.Haystack.alloc(n)
    hs.fill_synthetic(alphabet, seed)
    for pos, v in writes:
        hs.write(pos, v)
    return hs, pats, ks


def lists(res):
    return [res.arrays(w) for w in (F.RAW, F.FINAL)]


def same(a, b):
    return all(np.array_equal(x, y) for la, lb in zip(a, b) for x, y in zip(la, lb))


def measure(hs, pats, ks):
    warm, _ = hs.search_hamming_batch(pats[:64], ks[:64])  # warm-up: module load, pass buffers, byte statistics
    for r in warm:
        r.close()
    hs.timer_start()
    results, _ = hs.search_hamming_batch(pats, ks)
    got = [lists(r) for r in results]
    batch_ms = hs.timer_stop()
    stats = [r.stats() for r in results]
    for r in results:
        r.close()
    shared = [s for s in stats if s["route"] == SHARED]
    one = hs.search_hamming(pats[0], ks[0])  # warm-up of the single search
    one.close()
    single_ms, equal = 0.0, True
    for p, k, g in zip(pats, ks, got):
        hs.timer_start()
        one = hs.search_hamming(p, k)
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


def card():
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"],
                       capture_output=True, text=True, check=True).stdout.strip().splitlines()[0]
    name, power = [x.strip() for x in q.split(",")]
    return name, power


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--n", type=int, default=4 << 30)
    ap.add_argument("--patterns", type=int, default=1024)
    ap.add_argument("--workloads", default="dna,ascii")
    a = ap.parse_args()
    if F.device_count() == 0:
        raise SystemExit("no CUDA device")
    name, power = card()
    out = {"card": name, "power_limit": power, "n": a.n, "patterns": a.patterns}
    for w in a.workloads.split(","):
        hs, pats, ks = make_haystack(w, a.n, a.patterns)
        out[w] = measure(hs, pats, ks)
        hs.close()
    print(json.dumps(out))


if __name__ == "__main__":
    main()
