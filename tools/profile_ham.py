"""One Hamming search of 4 GiB of DNA (configs[2]) for ncu:
   ncu --set full --clock-control none --import-source on -k regex:k_hamming_count -c 1 \
       -o profiles/ham_sliced python tools/profile_ham.py"""
import os
import sys

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import numpy as np  # noqa: E402

from fuzzysearch_b200 import _native as F  # noqa: E402

n = int(sys.argv[1]) if len(sys.argv) > 1 else 4 << 30
dna = F.Haystack.alloc(n)
dna.fill_synthetic(b"ACGT", 20260930)
rng = np.random.default_rng(20260931)
a = np.frombuffer(b"ACGT", dtype=np.uint8)
p32 = bytes(a[rng.integers(0, 4, size=32)])
for _ in range(512):
    v = bytearray(p32)
    for _ in range(int(rng.integers(0, 5))):
        v[int(rng.integers(0, 32))] = int(a[rng.integers(0, 4)])
    dna.write(int(rng.integers(0, n - 32)), bytes(v))
r = dna.search_hamming(p32, 3)
print("matches", r.count(F.RAW), r.stats())
r.close()
dna.close()
