"""One pattern over many short sequences: a record set searched in one device pass against the same buffer without
records, against a per-sequence loop of find_near_matches, and against the reference (oracle/_ref, when built).

For each workload: the device time of the record-set search and of the same buffer searched without a record set
(fzb_timer, the two timed in turn, medians of --reps), the end-to-end time of find_near_matches_in_each from a Python list (join, upload,
search, Match lists), the per-sequence find_near_matches loop timed on the first --loop sequences and extrapolated,
the reference on one core (--ref-sample sequences) and on all cores (--ref-all-sample, workers started before the
clock), both extrapolated, and parity: the lists of the first --loop sequences equal this package's single searches
and a seeded sample of 200 equals the oracle.  Prints one JSON line per workload,
then one with the card's name and power limit.

    python tools/probe_records.py [--scale 1.0] [--reps 7] [--loop 10000] [--ref-sample 20000] [--ref-all-sample 400000]
"""
import argparse
import json
import multiprocessing
import os
import statistics
import subprocess
import sys
import time

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
import numpy as np

import oracle
from fuzzysearch_b200 import DeviceSequenceSet, _native as F, find_near_matches, find_near_matches_in_each

REF = os.path.join(ROOT, "oracle", "_ref")


def dna_reads(n, length=150, seed=7):
    rng = np.random.default_rng(seed)
    reads = np.frombuffer(b"ACGT", dtype=np.uint8)[rng.integers(0, 4, size=(n, length))]
    return rng, reads


def plant(rng, seqs, pat, alphabet, frac=0.05, edits=2):
    """a copy of `pat` with up to `edits` substitutions in `frac` of the sequences (a list of bytearrays)"""
    alpha = np.frombuffer(alphabet, dtype=np.uint8)
    for i in rng.choice(len(seqs), size=int(len(seqs) * frac), replace=False):
        v = bytearray(pat)
        for j in rng.integers(0, len(pat), size=int(rng.integers(0, edits + 1))):
            v[int(j)] = int(alpha[rng.integers(0, len(alpha))])
        s = seqs[i]
        if len(s) >= len(v):
            p = int(rng.integers(0, len(s) - len(v) + 1))
            s[p:p + len(v)] = v


def workloads(scale):
    n_reads, n_lines = int(1_000_000 * scale), int(2_000_000 * scale)
    rng, reads = dna_reads(n_reads)
    reads = [bytearray(r.tobytes()) for r in reads]
    p20 = bytes(np.frombuffer(b"ACGT", dtype=np.uint8)[rng.integers(0, 4, size=20)])
    p12 = bytes(np.frombuffer(b"ACGT", dtype=np.uint8)[rng.integers(0, 4, size=12)])
    plant(rng, reads, p20, b"ACGT")
    plant(rng, reads, p12, b"ACGT", edits=1)
    reads = [bytes(r) for r in reads]
    ascii_ = np.frombuffer(bytes(range(32, 127)), dtype=np.uint8)
    lens = rng.integers(40, 121, size=n_lines)
    flat = ascii_[rng.integers(0, len(ascii_), size=int(lens.sum()))].tobytes()
    ends = np.cumsum(lens)
    lines = [bytearray(flat[e - n:e]) for e, n in zip(ends.tolist(), lens.tolist())]
    p10 = bytes(ascii_[rng.integers(0, len(ascii_), size=10)])
    p8 = bytes(ascii_[rng.integers(0, len(ascii_), size=8)])
    plant(rng, lines, p10, bytes(range(32, 127)))
    plant(rng, lines, p8, bytes(range(32, 127)))
    lines = [bytes(x) for x in lines]
    generic = dict(max_substitutions=1, max_insertions=1, max_deletions=0, max_l_dist=2)
    return [("dna-reads/levenshtein-ngrams", reads, p20, dict(max_l_dist=2)),
            ("dna-reads/hamming", reads, p12, dict(max_substitutions=1, max_insertions=0, max_deletions=0)),
            ("ascii-lines/levenshtein-ngrams", lines, p10, dict(max_l_dist=2)),   # 10 // 3 >= 3: n-gram route
            ("ascii-lines/levenshtein-lp", lines, p8, dict(max_l_dist=2)),        # 8 // 3 < 3: LP route
            ("ascii-lines/generic-ngrams", lines, p10, generic),
            ("ascii-lines/generic-lp", lines, p8, generic)]


def device_search(hs, pat, lim):
    if lim.get("max_l_dist") == 2 and len(lim) == 1:
        return hs.search_levenshtein(pat, 2)
    if lim.get("max_insertions") == 0 and lim.get("max_deletions") == 0:
        return hs.search_hamming(pat, lim["max_substitutions"])
    return hs.search_generic(pat, lim["max_substitutions"], lim["max_insertions"], lim["max_deletions"],
                             lim["max_l_dist"])


def timed_once(hs, pat, lim):
    hs.timer_start()
    r = device_search(hs, pat, lim)
    r.count(F.FINAL)
    ms = hs.timer_stop()
    route = r.stats()["route"]
    r.close()
    return ms, route


def timed_alternating(hs, offsets, pat, lim, reps):
    """-> medians (ms) of the search with and without the record set, the two timed in turn on the same buffer (one
    warm-up of each first), and the routes they took"""
    times = {True: [], False: []}
    routes = {}
    for it in range(reps + 1):
        for rec in (True, False):
            hs.set_records(offsets if rec else None)
            ms, routes[rec] = timed_once(hs, pat, lim)
            if it:
                times[rec].append(ms)
    hs.set_records(offsets)
    return statistics.median(times[True]), statistics.median(times[False]), routes[True], routes[False]


_REF_JOB = None  # (pattern, sequences, limits) of the all-core run: the forked workers inherit it, nothing is pickled


def _ref_import():
    sys.path.insert(0, REF)
    import fuzzysearch  # noqa: F401


def _ref_run(pat, seqs, lim):
    _ref_import()
    import fuzzysearch as ref
    t0 = time.perf_counter()
    for s in seqs:
        ref.find_near_matches(pat, s, **lim)
    return time.perf_counter() - t0


def _ref_slice(part):
    pat, seqs, lim = _REF_JOB
    i, step, n = part
    return _ref_run(pat, seqs[i:n:step], lim)


def reference(pat, seqs, lim, n_one, n_all):
    """-> (single-core seconds, all-core seconds, cores) extrapolated to len(seqs) sequences, from the first n_one
    sequences on one core and the first n_all on every core (forked workers that have imported the reference before
    the clock starts), or None without oracle/_ref"""
    global _REF_JOB
    if not os.path.isdir(os.path.join(REF, "fuzzysearch")):
        return None
    n_one, n_all = min(n_one, len(seqs)), min(n_all, len(seqs))
    one = _ref_run(pat, seqs[:n_one], lim)
    cores = os.cpu_count() or 1
    _REF_JOB = (pat, seqs, lim)
    with multiprocessing.get_context("fork").Pool(cores, initializer=_ref_import) as pool:
        pool.map(_ref_slice, [(0, 1, 0)] * cores, chunksize=1)  # every worker up before the clock
        t0 = time.perf_counter()
        pool.map(_ref_slice, [(i, cores, n_all) for i in range(cores)], chunksize=1)
        allc = time.perf_counter() - t0
    _REF_JOB = None
    return one * len(seqs) / n_one, allc * len(seqs) / n_all, cores


def probe(name, seqs, pat, lim, args):
    out = {"workload": name, "sequences": len(seqs), "bytes": int(sum(len(s) for s in seqs)), "pattern_len": len(pat),
           "limits": lim}
    resident = DeviceSequenceSet(seqs)
    hs = resident._seq.haystack
    (out["device_ms_records"], out["device_ms_no_records"], out["route"],
     out["route_no_records"]) = timed_alternating(hs, resident.offsets, pat, lim, args.reps)
    out["records_over_plain"] = out["device_ms_records"] / out["device_ms_no_records"]
    resident.close()
    ends = []
    for _ in range(2):
        t0 = time.perf_counter()
        hits = find_near_matches_in_each(pat, seqs, **lim)
        ends.append(time.perf_counter() - t0)
    out["end_to_end_s"] = min(ends)
    out["matches"] = int(sum(len(h) for h in hits))
    loop = seqs[:args.loop]
    t0 = time.perf_counter()
    single = [find_near_matches(pat, s, **lim) for s in loop]
    t_loop = time.perf_counter() - t0
    out["loop_per_call_us"] = t_loop / len(loop) * 1e6
    out["loop_s_extrapolated"] = t_loop * len(seqs) / len(loop)
    out["parity_single_first_n"] = len(loop) if all(a == b for a, b in zip(hits, single)) else False
    rng = np.random.default_rng(1)
    sample = rng.choice(len(seqs), size=min(200, len(seqs)), replace=False)
    out["parity_oracle_sample"] = all(
        [(m.start, m.end, m.dist) for m in hits[i]] == [tuple(int(x) for x in r)
                                                        for r in oracle.find_near_matches(pat, seqs[i], **lim)]
        for i in sample.tolist())
    ref = reference(pat, seqs, lim, args.ref_sample, args.ref_all_sample)
    if ref:
        out["reference_single_core_s_extrapolated"], out["reference_all_cores_s_extrapolated"], out["cores"] = ref
    print(json.dumps(out), flush=True)
    return out


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--scale", type=float, default=1.0)
    ap.add_argument("--reps", type=int, default=7)
    ap.add_argument("--loop", type=int, default=10000)
    ap.add_argument("--ref-sample", type=int, default=20000)
    ap.add_argument("--ref-all-sample", type=int, default=400000)
    args = ap.parse_args()
    for w in workloads(args.scale):
        probe(*w, args)
    card = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                          capture_output=True, text=True).stdout.strip()
    print(json.dumps({"card": card}), flush=True)


if __name__ == "__main__":
    main()
