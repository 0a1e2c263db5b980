"""Levenshtein batches on DNA through the 2-bit n-gram pass (k_filter_mdense2 / k_verify_mhits), against one search per
pattern.

Workloads: (a) 4 GiB of synthetic ACGT on the device and 1 024 patterns of 15..40 symbols with max_l_dist 1..2 and
4 plants each: the batch against one search_levenshtein per pattern, both timed with the handle's device stopwatch
(fzb_timer, read-back included) in alternating rounds; the costs per posting and per verified hit (scan time beyond
the bare read of a two-pattern pass over the postings the pass walks, expected from the sampled byte statistics;
pass time beyond the scans over hits, which includes the host turnaround between chunks); the single search's cost
fitted as a per-search time plus a time per n-gram hit; the patterns with n-grams of 5 and of 6 symbols alone against
what they add to the batch (riding the pass or searched alone inside it, as admission decides); every list equal to its single search.  (b) About 1 M reads of 150 bases and 96 barcodes of
16..24 symbols at max_l_dist 1..2: find_near_matches_batch_in_each on a resident DeviceSequenceSet against a loop of
find_near_matches_in_each, end to end and on the device, and equal for every pattern and read.  Prints one JSON line
per workload, then the card's name and power limit (read in the same run).

    python tools/probe_dna_lev_batch.py [--gib 4] [--patterns 1024] [--reads 1000000] [--rounds 2]
"""
import argparse
import json
import os
import subprocess
import sys
import time

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
import numpy as np

from fuzzysearch_b200 import DeviceSequenceSet, _native as F, find_near_matches_batch_in_each, find_near_matches_in_each

DNA = b"ACGT"
DENSE = "ngrams/dense-filter"


def rand(rng, n):
    return bytes(np.frombuffer(DNA, dtype=np.uint8)[rng.integers(0, 4, size=n)])


def mutate(rng, p, e):
    v = bytearray(p)
    for _ in range(e):
        i = int(rng.integers(0, len(v)))
        op = int(rng.integers(0, 3))
        if op == 0:
            v[i] = DNA[int(rng.integers(0, 4))]
        elif op == 1 and len(v) > 1:
            del v[i]
        else:
            v.insert(i, DNA[int(rng.integers(0, 4))])
    return bytes(v)


def lists(r):
    return [a.copy() for a in r.arrays(F.RAW, anchors=True)] + [a.copy() for a in r.arrays(F.FINAL)]


def same(a, b):
    return len(a) == len(b) and all(np.array_equal(x, y) for x, y in zip(a, b))


def classify(stats, single_hits):
    """-> (first patterns of the passes, patterns in passes).  A pass reports its scan on its first pattern only, with
    the pass's hits; a pattern searched alone reports its own scan and hits (the single search's route is the same)."""
    heads = [q for q, s in enumerate(stats)
             if s["route"] == DENSE and s["bytes_scanned"] > 0 and s["n_candidates"] != single_hits[q]]
    shared = [q for q, s in enumerate(stats) if q in heads or (s["route"] == DENSE and s["bytes_scanned"] == 0)]
    return heads, shared


def postings_per_position(pats, ks, c=0.25):
    """expected postings walked per position by the 2-bit pass: n_ngrams * max(c, 1/4)^min(L, 8) per pattern"""
    tot = 0.0
    for p, k in zip(pats, ks):
        L = len(p) // (k + 1)
        tot += (len(p) // L) * max(c, 0.25) ** min(L, 8)
    return tot


def haystack_workload(args):
    rng = np.random.default_rng(41)
    n = int(args.gib * (1 << 30))
    hs = F.Haystack.alloc(n)
    hs.fill_synthetic(DNA, 43)
    pats = [rand(rng, int(m)) for m in rng.integers(15, 41, size=args.patterns)]
    ks = [int(k) for k in rng.integers(1, 3, size=args.patterns)]
    for p, k in zip(pats, ks):
        for _ in range(4):
            hs.write(int(rng.integers(0, n - 64)), mutate(rng, p, int(rng.integers(0, k + 1))))
    warm, _ = hs.search_levenshtein_batch(pats[:8], ks[:8])  # module load, pass buffers, byte statistics
    for r in warm:
        r.close()
    bare = [rand(rng, 40), rand(rng, 40)]  # two patterns with n-grams of 20 symbols: the scan is the read
    bare_res, bare_st = hs.search_levenshtein_batch(bare, [1, 1])
    bare_ms = bare_res[0].stats()["filter_ms"]
    for r in bare_res:
        r.close()
    out = {"workload": "dna%dg/lev-batch%d" % (args.gib, args.patterns), "bytes": n, "patterns": len(pats),
           "bare_scan_ms": round(bare_ms, 3)}
    batch_ms, single_ms, got, want = [], [], None, None
    for rnd in range(args.rounds):  # alternating arms
        hs.timer_start()
        res, total = hs.search_levenshtein_batch(pats, ks)
        g = [lists(r) for r in res]
        batch_ms.append(hs.timer_stop())
        stats = [r.stats() for r in res]
        for r in res:
            r.close()
        if got is None:
            got = g
        t = 0.0
        w, each_ms, each_hits = [], [], []
        for p, k in zip(pats, ks):
            hs.timer_start()
            one = hs.search_levenshtein(p, k)
            w.append(lists(one))
            each_ms.append(hs.timer_stop())
            each_hits.append(one.stats()["n_candidates"])
            t += each_ms[-1]
            one.close()
        single_ms.append(t)
        if want is None:
            want = w
    heads, shared = classify(stats, each_hits)
    # the single search's cost: time per search = a + b * its n-gram hits (least squares over the patterns)
    b_ms, a_ms = np.polyfit(np.array(each_hits, dtype=np.float64), np.array(each_ms), 1)
    # what the patterns with n-grams of 5 and of 6 symbols add to the batch (in the pass or alone, as admitted)
    lvals = [len(p) // (k + 1) for p, k in zip(pats, ks)]

    def batch_without(short):
        keep = [q for q in range(len(pats)) if lvals[q] > short]
        hs.timer_start()
        res, _ = hs.search_levenshtein_batch([pats[q] for q in keep], [ks[q] for q in keep])
        [lists(r) for r in res]
        ms = hs.timer_stop()
        for r in res:
            r.close()
        return ms

    without = {4: batch_ms[-1], 5: batch_without(5), 6: batch_without(6)}
    by_l = {}
    for L in (5, 6):
        qs = [q for q in range(len(pats)) if lvals[q] == L]
        by_l[L] = {"patterns": len(qs), "hits": int(sum(each_hits[q] for q in qs)),
                   "alone_ms": round(sum(each_ms[q] for q in qs), 1),
                   "riding": sum(1 for q in qs if q in shared),
                   "added_to_batch_ms": round(without[L - 1] - without[L], 1)}
    scans = [stats[q] for q in heads]
    scan_ms = sum(s["filter_ms"] for s in scans)
    hits = sum(s["n_candidates"] for s in scans)
    pass_ms = sum(s["gpu_ms"] for s in scans)
    post = postings_per_position([pats[q] for q in shared], [ks[q] for q in shared]) * n
    out.update({
        "batch_ms": [round(x, 1) for x in batch_ms], "one_by_one_ms": [round(x, 1) for x in single_ms],
        "batch_device_ms": round(total["gpu_ms"], 1), "passes": len(scans), "patterns_shared": len(shared),
        "patterns_one_by_one": len(pats) - len(shared), "pass_ms": round(pass_ms, 1), "scan_ms": round(scan_ms, 1),
        "hits": hits, "postings_expected": post,
        "ns_per_posting": (scan_ms - len(scans) * bare_ms) * 1e6 / post if post else None,
        "ns_per_hit": (pass_ms - scan_ms) * 1e6 / hits if hits else None,
        "single_fit": {"ms_per_search": round(a_ms, 3), "ns_per_hit": b_ms * 1e6},
        "by_L": by_l,
        "raw_matches": int(sum(len(x[0]) for x in got)),
        "equal_single": all(same(a, b) for a, b in zip(got, want)),
    })
    hs.close()
    return out


def reads_workload(args):
    rng = np.random.default_rng(42)
    acgt = np.frombuffer(DNA, dtype=np.uint8)
    reads = [bytearray(r.tobytes()) for r in acgt[rng.integers(0, 4, size=(args.reads, 150))]]
    codes = [rand(rng, int(m)) for m in rng.integers(16, 25, size=96)]
    ks = [1 + q % 2 for q in range(len(codes))]
    for c, k in zip(codes, ks):
        for i in rng.choice(len(reads), size=len(reads) // 100, replace=False):
            v = mutate(rng, c, int(rng.integers(0, k + 1)))
            p = int(rng.integers(0, 150 - len(v) + 1))
            reads[i][p:p + len(v)] = v
    reads = [bytes(r) for r in reads]
    resident = DeviceSequenceSet(reads)
    hs = resident._seq.haystack
    bound = resident._bind_many(codes)
    res, total = hs.search_levenshtein_batch(bound, ks, F.F_PER_RECORD)  # warm-up and routes
    stats = [r.stats() for r in res]
    for r in res:
        r.close()
    single_hits = []
    for c, k in zip(bound, ks):
        one = hs.search_levenshtein(c, k)
        single_hits.append(one.stats()["n_candidates"])
        one.close()
    heads, shared = classify(stats, single_hits)
    out = {"workload": "dna-reads%d/barcodes96-lev" % args.reads, "passes": len(heads),
           "patterns_shared": len(shared), "patterns_one_by_one": len(codes) - len(shared)}
    dev_b, dev_1, e2e_b, e2e_1 = [], [], [], []
    got = each = None
    for rnd in range(args.rounds):
        res, total = hs.search_levenshtein_batch(bound, ks, F.F_PER_RECORD)
        dev_b.append(total["gpu_ms"])
        for r in res:
            r.close()
        t = 0.0
        for c, k in zip(bound, ks):
            one = hs.search_levenshtein(c, k)
            t += one.stats()["gpu_ms"]
            one.close()
        dev_1.append(t)
        t0 = time.perf_counter()
        g = find_near_matches_batch_in_each(codes, resident, max_l_dist=ks)
        e2e_b.append(time.perf_counter() - t0)
        t0 = time.perf_counter()
        e = [find_near_matches_in_each(c, resident, max_l_dist=k) for c, k in zip(codes, ks)]
        e2e_1.append(time.perf_counter() - t0)
        if got is None:
            got, each = g, e
    out.update({
        "batch_device_ms": [round(x, 2) for x in dev_b], "one_by_one_device_ms": [round(x, 2) for x in dev_1],
        "batch_end_to_end_s": [round(x, 2) for x in e2e_b], "in_each_loop_s": [round(x, 2) for x in e2e_1],
        "matches": int(sum(len(ms) for d in got for ms in d.values())),
        "equal_in_each": all(got[q] == {r: ms for r, ms in enumerate(e) if ms} for q, e in enumerate(each)),
    })
    resident.close()
    return out


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--gib", type=float, default=4)
    ap.add_argument("--patterns", type=int, default=1024)
    ap.add_argument("--reads", type=int, default=1_000_000)
    ap.add_argument("--rounds", type=int, default=2)
    ap.add_argument("--only", choices=("haystack", "reads"))
    args = ap.parse_args()
    card = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                          capture_output=True, text=True).stdout.strip()
    if args.only in (None, "haystack"):
        print(json.dumps(haystack_workload(args)), flush=True)
    if args.only in (None, "reads"):
        print(json.dumps(reads_workload(args)), flush=True)
    print(json.dumps({"card": card}), flush=True)


if __name__ == "__main__":
    main()
