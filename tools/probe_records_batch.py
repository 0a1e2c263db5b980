"""Many patterns over many short sequences: batches with FZB_F_PER_RECORD on a resident record set, against the same
batches on the same buffer without the record set, and against a loop of find_near_matches_in_each (one call per
pattern).

Workloads: (a) DNA reads of 150 bytes and 96 barcodes of 8..24 bytes with 1..2 substitutions (demultiplexing);
(b) ASCII lines of 40..120 bytes (the generator of tools/probe_records.py) and 1 024 terms of 8..64 bytes with a mix
of Levenshtein, substitutions-only and generic limits.  For each: the device time of the batch with and without the
record set (the summed pass and search times the batch reports, the two timed in turn, medians of --reps), the
end-to-end time of find_near_matches_batch_in_each on the resident set, the find_near_matches_in_each loop over the first --loop patterns (extrapolated to all), how many
patterns rode on shared scans (per route: patterns, scans), and parity: for every looped pattern, its entries for the first
10 000 records equal its find_near_matches_in_each.  Prints one JSON line per workload, then the card's name and
power limit.

    python tools/probe_records_batch.py [--scale 1.0] [--reps 5] [--loop 96] [--only dna|ascii]
"""
import argparse
import json
import os
import statistics
import subprocess
import sys
import time

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
import numpy as np

from fuzzysearch_b200 import (DeviceSequenceSet, _batch_params, _native as F, find_near_matches_batch_in_each,
                              find_near_matches_in_each)
from fuzzysearch_b200.search import ExactSearch, GenericSearch, LevenshteinSearch, SubstitutionsOnlySearch

PARITY_RECORDS = 10_000


def plant(rng, seqs, pat, alphabet, frac, edits):
    alpha = np.frombuffer(alphabet, dtype=np.uint8)
    for i in rng.choice(len(seqs), size=max(1, int(len(seqs) * frac)), replace=False):
        v = bytearray(pat)
        for j in rng.integers(0, len(pat), size=int(rng.integers(0, edits + 1))):
            v[int(j)] = int(alpha[rng.integers(0, len(alpha))])
        s = seqs[i]
        if len(s) >= len(v):
            p = int(rng.integers(0, len(s) - len(v) + 1))
            s[p:p + len(v)] = v


def dna_workload(scale):
    rng = np.random.default_rng(17)
    n = int(1_000_000 * scale)
    acgt = np.frombuffer(b"ACGT", dtype=np.uint8)
    reads = [bytearray(r.tobytes()) for r in acgt[rng.integers(0, 4, size=(n, 150))]]
    codes = [bytes(acgt[rng.integers(0, 4, size=int(m))]) for m in rng.integers(8, 25, size=96)]
    subs = [1 + q % 2 for q in range(len(codes))]
    for c, k in zip(codes, subs):
        plant(rng, reads, c, b"ACGT", 0.01, k)
    return [bytes(r) for r in reads], codes, dict(max_substitutions=subs, max_insertions=0, max_deletions=0)


def ascii_workload(scale):
    rng = np.random.default_rng(18)
    n = int(2_000_000 * scale)
    ascii_ = np.frombuffer(bytes(range(32, 127)), dtype=np.uint8)
    lens = rng.integers(40, 121, size=n)
    flat = ascii_[rng.integers(0, len(ascii_), size=int(lens.sum()))].tobytes()
    ends = np.cumsum(lens)
    lines = [bytearray(flat[e - m:e]) for e, m in zip(ends.tolist(), lens.tolist())]
    terms = [bytes(ascii_[rng.integers(0, len(ascii_), size=int(m))]) for m in rng.integers(8, 65, size=1024)]
    subs, ins, dels, ls = [], [], [], []
    for q, t in enumerate(terms):
        k = 1 if len(t) < 16 else 2
        kind = q % 3  # Levenshtein, substitutions-only, generic
        subs.append(k)
        ins.append(0 if kind == 1 else (k if kind == 0 else 1))
        dels.append(0 if kind == 1 else (k if kind == 0 else 0))
        ls.append(k)
        plant(rng, lines, t, bytes(range(32, 127)), 0.0005, k)
    lines = [bytes(x) for x in lines]
    return lines, terms, dict(max_substitutions=subs, max_insertions=ins, max_deletions=dels, max_l_dist=ls)


def batches(hs, pats, params, classes, flags):
    """the three class batches of find_near_matches_batch_in_each -> (summed device ms, results)"""
    n = len(pats)
    lev = [i for i in range(n) if classes[i] in (ExactSearch, LevenshteinSearch)]
    ham = [i for i in range(n) if classes[i] is SubstitutionsOnlySearch]
    gen = [i for i in range(n) if classes[i] is GenericSearch]
    ms, results = 0.0, []
    if lev:
        rs, st = hs.search_levenshtein_batch([pats[i] for i in lev], [params[i].max_l_dist for i in lev], flags)
        ms += st["gpu_ms"]
        results += rs
    if ham:
        ks = [min(x for x in (params[i].max_l_dist, params[i].max_substitutions) if x is not None) for i in ham]
        rs, st = hs.search_hamming_batch([pats[i] for i in ham], ks, flags)
        ms += st["gpu_ms"]
        results += rs
    if gen:
        rs, st = hs.search_generic_batch([pats[i] for i in gen], *zip(*[params[i].unpacked for i in gen]), flags=flags)
        ms += st["gpu_ms"]
        results += rs
    return ms, results


def routes(results):
    """route -> [patterns, scans]; a route with more patterns than scans shared them"""
    out = {}
    for r in results:
        st = r.stats()
        e = out.setdefault(st["route"], [0, 0])
        e[0] += 1
        e[1] += st["bytes_scanned"] > 0
    return out


def probe(name, seqs, pats, lim, reps, loop):
    out = {"workload": name, "sequences": len(seqs), "bytes": int(sum(len(s) for s in seqs)), "patterns": len(pats)}
    _, _, params, classes = _batch_params(pats, lim.get("max_substitutions"), lim.get("max_insertions"),
                                          lim.get("max_deletions"), lim.get("max_l_dist"))
    resident = DeviceSequenceSet(seqs)
    hs = resident._seq.haystack
    bound = resident._bind_many(pats)
    times = {True: [], False: []}
    for it in range(reps + 1):
        for rec in (True, False):
            hs.set_records(resident.offsets if rec else None)
            ms, results = batches(hs, bound, params, classes, F.F_PER_RECORD if rec else 0)
            if rec:
                out["routes_records"] = routes(results)
            else:
                out["routes_no_records"] = routes(results)
            for r in results:
                r.close()
            if it:
                times[rec].append(ms)
    hs.set_records(resident.offsets)
    out["device_ms_records"] = statistics.median(times[True])
    out["device_ms_no_records"] = statistics.median(times[False])
    t0 = time.perf_counter()
    got = find_near_matches_batch_in_each(pats, resident, **lim)
    out["end_to_end_s"] = time.perf_counter() - t0
    out["matches"] = int(sum(len(ms) for d in got for ms in d.values()))
    t0 = time.perf_counter()
    ok = True
    n_loop = min(loop, len(pats))
    for q, p in enumerate(pats[:n_loop]):
        one = {k: (v[q] if isinstance(v, list) else v) for k, v in lim.items()}
        each = find_near_matches_in_each(p, resident, **one)
        ok &= all(got[q].get(r, []) == each[r] for r in range(min(PARITY_RECORDS, len(seqs))))
        if q % 16 == 15:
            print("  %s: %d of %d patterns looped" % (name, q + 1, n_loop), file=sys.stderr, flush=True)
    out["loop_in_each_patterns"] = n_loop
    out["loop_in_each_s"] = time.perf_counter() - t0
    out["loop_in_each_s_extrapolated"] = out["loop_in_each_s"] * len(pats) / n_loop
    out["parity_first_10000_records"] = ok
    resident.close()
    return out


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--scale", type=float, default=1.0)
    ap.add_argument("--reps", type=int, default=5)
    ap.add_argument("--loop", type=int, default=96, help="patterns of the find_near_matches_in_each loop (the rest "
                                                           "extrapolated) and of the parity check")
    ap.add_argument("--only", choices=("dna", "ascii"))
    args = ap.parse_args()
    card = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"],
                          capture_output=True, text=True).stdout.strip()
    if args.only in (None, "dna"):
        reads, codes, lim = dna_workload(args.scale)
        print(json.dumps(probe("dna-reads/barcodes-hamming", reads, codes, lim, args.reps, args.loop)), flush=True)
        del reads
    if args.only in (None, "ascii"):
        lines, terms, lim = ascii_workload(args.scale)
        print(json.dumps(probe("ascii-lines/terms-mixed", lines, terms, lim, args.reps, args.loop)), flush=True)
    print(json.dumps({"card": card}), flush=True)


if __name__ == "__main__":
    main()
