"""Measure the sampled scan (k_filter_sampled) of the bench workload against a plain read of the same buffer, and
break one search into its kernels.  Prints one JSON line.  Measurement only: bench.py and the tests do not use it.

    python tools/probe_scan.py [--n BYTES] [--searches 30]
    python tools/probe_scan.py --ab OTHER/libfuzzb200.so [--rounds 5]

* card: name, power limit and max SM clock (read-only nvidia-smi query).
* read reference: torch sum over the resident haystack buffer viewed as int64 (a torch read-only reduction, not a
  peak).
* scan: filter_ms (the CUDA events around k_filter_sampled) of `--searches` searches after warm-up.
* step: device ms per search (the events around the whole loop, as bench.py times it) and host wall ms per search.
* trace: one torch.profiler pass of a few searches: per-kernel durations, the gaps between k_filter_sampled,
  k_verify_lev and k_post, and the phase times of k_post's last CTA (debug_counters()[10:14]).
* --ab: the same searches on this package's library and on another build of it, in alternating rounds; both series.
"""
import argparse
import ctypes
import json
import os
import statistics
import subprocess
import sys
import time

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import numpy as np

import bench
from fuzzysearch_b200 import _native as F

M, K, SEED = 20, 2, 20260923


def card():
    try:
        out = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                             capture_output=True, text=True, timeout=30).stdout.strip().splitlines()
        name, power, clock = [x.strip() for x in out[0].split(",")]
        return {"name": name, "power_limit": power, "max_sm_clock": clock}
    except Exception as e:  # the numbers below still stand, without the card they were taken on
        return {"error": str(e)}


def load(path):
    """A second build of the library, with the same symbol table as the package's."""
    lib = ctypes.CDLL(os.path.abspath(path))
    for name, (res, args) in F.SYMBOLS.items():
        f = getattr(lib, name)
        f.restype, f.argtypes = res, args
    return lib


def make_haystack(n):
    alphabet = bench.ASCII
    hs = F.Haystack.alloc(n)
    hs.fill_synthetic(alphabet, SEED)
    rng = np.random.default_rng(SEED)
    pat = bytes(np.frombuffer(alphabet, dtype=np.uint8)[rng.integers(0, len(alphabet), size=M)])
    for pos, b in bench.make_plants(SEED + 1, 0, n, M, K, pat, alphabet, 4096, False):
        hs.write(pos, b)
    return hs, pat


def one(hs, pat):
    r = hs.search_levenshtein(pat, K)
    st = r.stats()
    nf = r.count(F.FINAL)
    r.close()
    return st, nf


def series(hs, pat, searches):
    """filter_ms of each search, device ms per search of the loop, wall ms per search, final count."""
    filt = []
    hs.timer_start()
    t0 = time.perf_counter()
    for _ in range(searches):
        st, nf = one(hs, pat)
        filt.append(st["filter_ms"])
    dev = hs.timer_stop() / searches
    wall = (time.perf_counter() - t0) * 1e3 / searches
    return filt, dev, wall, nf


def summary(xs):
    xs = sorted(xs)
    return {"median": statistics.median(xs), "min": xs[0], "max": xs[-1]}


def torch_read(hs, n, reps=20):
    import torch

    class View:  # the haystack's device buffer as int64 (n is a multiple of 8)
        __cuda_array_interface__ = {"shape": (n // 8,), "typestr": "<i8", "data": (hs.dev_ptr, False), "version": 2}

    t = torch.as_tensor(View(), device="cuda")
    for _ in range(3):
        t.sum()
    torch.cuda.synchronize()
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    ms = []
    for _ in range(reps):
        e0.record()
        t.sum()
        e1.record()
        e1.synchronize()
        ms.append(e0.elapsed_time(e1))
    s = summary(ms)
    return {"what": "torch read-only reduction (int64 sum) over the haystack buffer", "ms": s,
            "GB_per_s": n / (s["median"] * 1e-3) / 1e9}


def trace(hs, pat, searches=5):
    import torch
    from torch.profiler import ProfilerActivity, profile

    with profile(activities=[ProfilerActivity.CPU, ProfilerActivity.CUDA]) as prof:
        for _ in range(searches):
            one(hs, pat)
        torch.cuda.synchronize()
    kern = sorted((e for e in prof.events() if e.device_type == torch.autograd.DeviceType.CUDA),
                  key=lambda e: e.time_range.start)
    per_kernel, gaps = {}, {}
    prev = None
    for e in kern:
        name = e.name.split("(")[0].split("<")[0].replace("fzb::", "").replace("void ", "")
        per_kernel.setdefault(name, []).append((e.time_range.end - e.time_range.start) / 1e3)
        if prev is not None:
            gaps.setdefault(prev[0] + " -> " + name, []).append((e.time_range.start - prev[1]) / 1e3)
        prev = (name, e.time_range.end)
    cn = hs.debug_counters()
    return {"kernel_ms": {k: summary(v) for k, v in per_kernel.items()},
            "gap_ms": {k: summary(v) for k, v in gaps.items()},
            "k_post_last_cta_ns": {"rank": cn[10], "ticket": cn[11], "sweep": cn[12], "copy": cn[13]}}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--n", type=int, default=4 << 30, help="haystack bytes (default 4 GiB, the bench workload)")
    ap.add_argument("--searches", type=int, default=30)
    ap.add_argument("--warmup", type=int, default=5)
    ap.add_argument("--ab", metavar="LIB", help="another build of libfuzzb200.so to alternate with")
    ap.add_argument("--rounds", type=int, default=5)
    args = ap.parse_args()
    n = args.n
    out = {"card": card(), "bytes": n, "workload": "find_near_matches(|pattern|=%d, ASCII, max_l_dist=%d)" % (M, K)}

    libs = [("this", F.lib())]
    if args.ab:
        libs.append((args.ab, load(args.ab)))
    setups = []
    for name, lib in libs:
        F._lib = lib
        hs, pat = make_haystack(n)
        for _ in range(args.warmup):
            one(hs, pat)
        setups.append((name, lib, hs, pat))
    F._lib = libs[0][1]
    out["read_reference"] = torch_read(setups[0][2], n)

    runs = {name: [] for name, *_ in setups}
    for _ in range(args.rounds if args.ab else 1):
        for name, lib, hs, pat in setups:
            F._lib = lib
            filt, dev, wall, nf = series(hs, pat, args.searches)
            fm = statistics.median(filt)
            runs[name].append({"filter_ms": summary(filt), "filter_GB_per_s": n / (fm * 1e-3) / 1e9,
                               "gpu_ms_per_search": dev, "wall_ms_per_search": wall, "final": nf})
    out["runs"] = runs
    if args.ab:
        out["ms_per_search"] = {name: summary([r["gpu_ms_per_search"] for r in rs]) for name, rs in runs.items()}
        out["filter_ms_median"] = {name: summary([r["filter_ms"]["median"] for r in rs]) for name, rs in runs.items()}
    F._lib = libs[0][1]
    out["trace"] = trace(setups[0][2], setups[0][3])
    for _, lib, hs, _ in setups:
        F._lib = lib
        hs.close()
    F._lib = libs[0][1]
    print(json.dumps(out))


if __name__ == "__main__":
    main()
