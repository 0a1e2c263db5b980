"""One invocation of every hot kernel on the 4 GiB workloads, for ncu:
   ncu --set full --clock-control none --import-source on -k regex:'k_(filter|verify|post|hamming|lp_|merge|push)' \
       -o profiles/all_kernels python tools/profile_all.py"""
import os
import sys

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import numpy as np

import bench
from fuzzysearch_b200 import _native as F

n = int(sys.argv[1]) if len(sys.argv) > 1 else 4 << 30
reps = int(sys.argv[2]) if len(sys.argv) > 2 else 1
seed = 20260923
rng = np.random.default_rng(seed)
# --- ASCII: headline search, LP search, 1024-pattern batch ------------------------------------------------
hs = F.Haystack.alloc(n)
hs.fill_synthetic(bench.ASCII, seed)
alpha = np.frombuffer(bench.ASCII, dtype=np.uint8)
pat = bytes(alpha[rng.integers(0, len(alpha), size=20)])
for pos, b in bench.make_plants(seed + 1, 0, n, 20, 2, pat, bench.ASCII, 4096, False):
    hs.write(pos, b)
for _ in range(reps):
    hs.search_levenshtein(pat, 2).close()                      # k_filter_sampled, k_verify_lev, k_post
    hs.search_levenshtein(pat[:9], 3).close()                  # k_lp_scan, k_lp_verify (m // (k+1) = 2: LP route)
brng = np.random.default_rng(seed + 99)
pats, ks = [], []
for i in range(1024):
    bm, bk = int(brng.integers(8, 65)), int(brng.integers(1, 5))
    bp = bytes(alpha[brng.integers(0, len(alpha), size=bm)])
    pats.append(bp)
    ks.append(bk)
    for _ in range(8):
        hs.write(1000 + int(brng.integers(0, n - 2000)), bench.mutate(brng, bp, bench.ASCII, int(brng.integers(0, bk + 2)), False))
for _ in range(reps):
    res, _ = hs.search_levenshtein_batch(pats, ks)             # k_filter_multi/k_verify_multi, k_filter_mdense/
    for r in res:                                              # k_verify_mhits, k_lp_scan_multi/k_lm_*/k_lp_verify_multi
        r.close()
hs.close()
# --- DNA: Hamming (TMA counting filter) and Levenshtein (dense filter + hit list) -----------------------------
dna = F.Haystack.alloc(n)
dna.fill_synthetic(bench.DNA, seed + 7)
a = np.frombuffer(bench.DNA, dtype=np.uint8)
p32 = bytes(a[rng.integers(0, 4, size=32)])
p20 = bytes(a[rng.integers(0, 4, size=20)])
for pos, b in bench.make_plants(seed + 8, 0, n, 32, 3, p32, bench.DNA, 4096, True):
    dna.write(pos, b)
for _ in range(reps):
    dna.search_hamming(p32, 3).close()                         # k_hamming_count, k_verify_ham
    dna.search_levenshtein(p20, 2).close()                     # k_filter_dense2, k_verify_hits
dna.close()
print("done")
