"""fzb_search_hamming_batch: many substitutions-only patterns over one resident haystack in shared scans
(k_ham_batch_scan, DESIGN.md section 5.8), and find_near_matches_batch with per-pattern limits of every search class.
Every case checks that each pattern's lists equal the single search_hamming on the same handle (RAW, FINAL, counts),
the oracle where the size allows, and that exactly the expected patterns took a shared pass."""
import os
import sys

import numpy as np
import pytest

import oracle
from conftest import needs_real_gpu
from corpus import ASCII, DNA
from fuzzysearch_b200 import DeviceSequence, _native as F, find_near_matches, find_near_matches_batch
from parity import tup

pytestmark = pytest.mark.gpu

SHARED, SINGLE = "hamming/batch-scan", "hamming"


def rand_bytes(rng, alphabet, m):
    alpha = np.frombuffer(alphabet, dtype=np.uint8)
    return bytes(alpha[rng.integers(0, len(alpha), size=m)])


def substitute(rng, pat, alphabet, e):
    """`pat` with e distinct positions replaced by a different symbol"""
    v = bytearray(pat)
    for i in rng.choice(len(v), size=min(e, len(v)), replace=False):
        v[i] = next(c for c in rng.permutation(np.frombuffer(alphabet, dtype=np.uint8)) if c != v[i])
    return bytes(v)


def plant(hay, pos, v):
    v = v[:len(hay) - pos]
    hay[pos:pos + len(v)] = np.frombuffer(v, dtype=np.uint8)


def plant_all(rng, hay, pats, ks, alphabet, per=3):
    """`per` copies of each pattern with 0..k substitutions and one with k+1"""
    n = len(hay)
    for p, k in zip(pats, ks):
        for e in [int(rng.integers(0, k + 1)) for _ in range(per)] + [k + 1]:
            plant(hay, int(rng.integers(0, max(1, n - len(p)))), substitute(rng, p, alphabet, e))


def check(hs, pats, ks, results, shared, hay=None):
    """Each result equals the single search on `hs`; with `hay` (the whole sequence) also the oracle; the patterns
    flagged in `shared`, and only those, took a shared pass."""
    assert len(results) == len(pats)
    for i, (p, k, r) in enumerate(zip(pats, ks, results)):
        assert r.stats()["route"] == (SHARED if shared[i] else SINGLE), (i, len(p), k)
        one = hs.search_hamming(p, k)
        for w in (F.RAW, F.FINAL):
            assert r.count(w) == one.count(w), (i, len(p), k, w)
            assert r.triples(w) == one.triples(w), (i, len(p), k, w)
        one.close()
        if hay is not None and k < len(p):
            assert r.triples(F.RAW) == tup(oracle.substitutions(p, bytes(hay), k)), (i, len(p), k)


def passes(results):
    """number of shared scans (a shared pass reports its scan on its first pattern only)"""
    return sum(1 for r in results if r.stats()["route"] == SHARED and r.stats()["bytes_scanned"] > 0)


def close_all(results):
    for r in results:
        r.close()


def dna_mix(rng):
    """-> (patterns, ks, shared?) on a DNA haystack: 2-bit keys need L = m // (k+1) >= 5"""
    pats, ks, shared = [], [], []
    for m, k, s in [(20, 3, True), (24, 2, True), (32, 1, True), (27, 3, True), (21, 0, True), (64, 7, True),
                    (70, 2, False),   # m > 64
                    (6, 6, False),    # k >= m
                    (12, 2, False),   # L = 4: key too short
                    (19, 3, False)]:  # L = 4
        pats.append(rand_bytes(rng, DNA, m))
        ks.append(k)
        shared.append(s)
    pats.append(pats[0][:10] + b"N" + pats[0][11:])  # an N inside a pattern (the code table aliases a byte)
    ks.append(3)
    shared.append(True)
    return pats, ks, shared


def ascii_mix(rng):
    """-> (patterns, ks, shared?) on text: keys of min(L, 4) bytes, one pass for 4-byte keys and one for 3-byte keys
    (L = 3); L = 2 is too short"""
    pats, ks, shared = [], [], []
    for m, k, s in [(12, 1, True), (20, 4, True), (64, 3, True), (33, 2, True), (16, 0, True), (8, 1, True),
                    (65, 1, False), (10, 10, False), (12, 3, True), (19, 4, True), (17, 4, True),
                    (14, 4, False), (11, 3, False)]:
        pats.append(rand_bytes(rng, ASCII, m))
        ks.append(k)
        shared.append(s)
    return pats, ks, shared


def dna_haystack(rng, n, n_runs=6):
    hay = np.frombuffer(rand_bytes(rng, DNA, n), dtype=np.uint8).copy()
    for _ in range(n_runs):  # runs of N: alias to some code of the 2-bit keys
        pos = int(rng.integers(0, n - 100))
        hay[pos:pos + int(rng.integers(10, 90))] = ord("N")
    return hay


def test_dna_and_ascii_mixes(cuda_device):
    rng = np.random.default_rng(8101)
    for alphabet, n, mix, npasses in ((DNA, 30000, dna_mix, 1), (ASCII, 30000, ascii_mix, 2)):
        pats, ks, shared = mix(rng)
        hay = dna_haystack(rng, n) if alphabet == DNA else np.frombuffer(rand_bytes(rng, ASCII, n), np.uint8).copy()
        plant_all(rng, hay, pats, ks, alphabet)
        hs = F.Haystack.from_host(hay)
        for _ in range(2):  # twice on the same handle
            rs, total = hs.search_hamming_batch(pats, ks)
            check(hs, pats, ks, rs, shared, hay=hay)
            assert passes(rs) == npasses
            assert sum(r.count(F.RAW) for r in rs) >= 3 * len(pats)
            close_all(rs)
        hs.close()


def test_two_bit_keys_on_wide_symbols(cuda_device):
    """A str of four symbols outside latin-1 is reduced to bytes 1..4 on the device: the 2-bit keys must tell them
    apart.  A fixed (c >> 1) & 3 would map 2 and 3 to one code; the verification would still drop the extra
    candidates, so the test bounds the candidates the shared pass verified by twice the expected number (random
    piece hits plus the planted copies); with codes 0, 1, 1, 2 a 5-symbol key hits about 7.6 times as often."""
    rng = np.random.default_rng(8102)
    sym = "αβγδ"
    text = "".join(sym[i] for i in rng.integers(0, 4, size=20000))
    pats = ["".join(sym[i] for i in rng.integers(0, 4, size=m)) for m in (20, 24, 30, 40)]
    ks = [3, 2, 2, 4]
    for p, k in zip(pats, ks):
        for _ in range(3):
            pos = int(rng.integers(0, len(text) - len(p)))
            text = text[:pos] + p + text[pos + len(p):]
    ds = DeviceSequence(text)
    bound = ds._bind_many(pats)
    hay = np.frombuffer(ds.haystack.read(0, len(text)), dtype=np.uint8)
    assert set(hay.tolist()) == {1, 2, 3, 4}
    rs, _ = ds.haystack.search_hamming_batch(bound, ks)
    check(ds.haystack, bound, ks, rs, [True] * 4, hay=hay)
    assert all(r.count(F.RAW) >= 3 for r in rs)
    expected = sum((k + 1) * (len(text) * 0.25 ** min(len(p) // (k + 1), 8) + 3) for p, k in zip(pats, ks))
    assert passes(rs) == 1 and sum(r.stats()["n_candidates"] for r in rs) <= 2 * expected
    close_all(rs)
    got = find_near_matches_batch(pats, ds, max_substitutions=ks, max_insertions=0, max_deletions=0)
    assert got == [find_near_matches(p, text, max_substitutions=k, max_insertions=0, max_deletions=0)
                   for p, k in zip(pats, ks)]
    ds.close()


def test_each_start_exactly_once(cuda_device):
    """Starts where every piece matches exactly, periodic patterns whose pieces occur at many offsets, duplicate
    patterns and patterns that are prefixes of each other in one pass, matches at 0 and at N - m."""
    rng = np.random.default_rng(8103)
    n = 20000
    hay = np.frombuffer(rand_bytes(rng, DNA, n), dtype=np.uint8).copy()
    p = rand_bytes(rng, DNA, 24)
    for pos in (0, 500, 530, 7000, n - 24):  # exact copies: all k+1 pieces match
        plant(hay, pos, p)
    plant(hay, 3000, b"AC" * 150)
    plant(hay, 9000, b"A" * 120)
    pats = [p, p, p[:20], p[:22], b"AC" * 12, b"CA" * 15, b"A" * 20, substitute(rng, p, DNA, 2)]
    ks = [3, 2, 3, 1, 2, 1, 3, 3]
    hs = F.Haystack.from_host(hay)
    for _ in range(2):
        rs, _ = hs.search_hamming_batch(pats, ks)
        check(hs, pats, ks, rs, [True] * len(pats), hay=hay)
        starts = [r.arrays(F.RAW)[0] for r in rs]
        assert all(np.all(np.diff(s) > 0) for s in starts)  # ascending, no start twice
        assert {0, 500, 530, 7000, n - 24} <= set(starts[0].tolist())
        assert len(starts[4]) >= 130 and len(starts[6]) >= 100
        close_all(rs)
    hs.close()
    # a pattern longer than the sequence
    short = np.frombuffer(b"ACGTACGTTGCAACGTACGTTGCAAC", dtype=np.uint8).copy()
    hs = F.Haystack.from_host(short)
    pats = [rand_bytes(rng, DNA, 40), bytes(short[:20]), bytes(short[3:23])]
    ks = [2, 1, 3]
    rs, _ = hs.search_hamming_batch(pats, ks)
    check(hs, pats, ks, rs, [True] * 3, hay=short)
    assert rs[0].count(F.RAW) == 0 and rs[1].count(F.RAW) >= 1
    close_all(rs)
    hs.close()


def test_batch_at_64_bit_offsets(cuda_device):
    """The same bytes as an interior shard at global offsets 0 .. 2^44: the batch at each offset is the batch at 0,
    shifted."""
    rng = np.random.default_rng(8104)
    n = 30000
    hay = dna_haystack(rng, n)
    pats, ks, shared = dna_mix(rng)
    plant_all(rng, hay, pats, ks, DNA)
    lo, hi = 256, n - 256
    a = F.Haystack.from_host(hay, buf_lo=0, global_len=n + (1 << 20), own_lo=lo, own_hi=hi)
    ra, _ = a.search_hamming_batch(pats, ks)
    check(a, pats, ks, ra, shared)
    assert sum(r.count(F.RAW) for r in ra) >= 2 * len(pats)
    for shift in (1 << 32, (1 << 40) + 16 * 12345, 1 << 44):
        b = F.Haystack.from_host(hay, buf_lo=shift, global_len=shift + n + (1 << 20), own_lo=shift + lo,
                                 own_hi=shift + hi)
        rb, _ = b.search_hamming_batch(pats, ks)
        for x, y in zip(ra, rb):
            assert y.stats()["route"] == x.stats()["route"]
            for w in (F.RAW, F.FINAL):
                assert [(s + shift, e + shift, d) for s, e, d in x.triples(w)] == y.triples(w), hex(shift)
        close_all(rb)
        b.close()
    close_all(ra)
    a.close()


@pytest.mark.parametrize("nshards", [2, 3, 7])
def test_sharded_union_equals_whole(cuda_device, nshards):
    """A batch on each shard (halo = the longest pattern): the union of the shards' lists is the whole handle's
    batch, with near-matches straddling every seam.  A pattern longer than the halo fails the batch on a shard with
    the single search's error."""
    rng = np.random.default_rng(8200 + nshards)
    n = (1 << 16) + 5
    hay = dna_haystack(rng, n)
    pats, ks, shared = dna_mix(rng)
    plant_all(rng, hay, pats, ks, DNA)
    bounds = [((n * i // nshards) // 16) * 16 for i in range(nshards)] + [n]
    for si, b in enumerate(bounds[1:-1]):
        for j, delta in enumerate((-1, -5, -12, 1)):
            q = (si + j) % len(pats)
            m = len(pats[q])
            plant(hay, b + delta - m // 2 + 200 * j, substitute(rng, pats[q], DNA, min(ks[q], 1)))
    whole = F.Haystack.from_host(hay)
    rw, _ = whole.search_hamming_batch(pats, ks)
    check(whole, pats, ks, rw, shared, hay=hay)
    halo = max(len(p) for p in pats)
    union = [[] for _ in pats]
    for i in range(nshards):
        lo, hi = bounds[i], bounds[i + 1]
        blo = max(0, lo - halo) // 16 * 16
        bhi = min(n, hi + halo)
        hs = F.Haystack.from_host(hay[blo:bhi], buf_lo=blo, global_len=n, own_lo=lo, own_hi=hi)
        rs, _ = hs.search_hamming_batch(pats, ks)
        check(hs, pats, ks, rs, shared)
        for q, r in enumerate(rs):
            union[q] += r.triples(F.RAW)
        close_all(rs)
        big = rand_bytes(rng, DNA, halo + 20)
        with pytest.raises(ValueError) as single:
            hs.search_hamming(big, 2)
        with pytest.raises(ValueError) as batch:
            hs.search_hamming_batch(pats + [big], ks + [2])
        assert str(batch.value) == str(single.value)
        hs.close()
    for q, r in enumerate(rw):
        assert sorted(union[q]) == r.triples(F.RAW), q
    close_all(rw)
    whole.close()


def test_pass_limits(cuda_device):
    """Patterns beyond one pass's bound on expected postings (two passes), a key with more postings than one table
    slot holds, and an FZB_F_TINY_LIST overflow (the pass's patterns go one by one) followed by a normal batch on the
    same handle.  Every scenario runs twice on the same handle."""
    rng = np.random.default_rng(8105)
    n = 12000
    hay = np.frombuffer(rand_bytes(rng, DNA, n), dtype=np.uint8).copy()
    # 70 patterns of m = 20, k = 3: four 5-symbol pieces each, about 4 / 4^5 expected postings per position
    many = [rand_bytes(rng, DNA, 20) for _ in range(70)]
    many_k = [3] * len(many)
    plant_all(rng, hay, many[:10], many_k[:10], DNA, per=1)
    # 33 copies of a period-8 pattern with k = 7: eight identical pieces -> 264 postings under one key
    per8 = b"ACGTTGCA" * 8
    plant(hay, 4000, per8)
    plant(hay, 6000, substitute(rng, per8, DNA, 5))
    dup = [per8] * 33
    dup_k = [7] * 33
    hs = F.Haystack.from_host(hay)
    for _ in range(2):
        rs, _ = hs.search_hamming_batch(many, many_k)
        check(hs, many, many_k, rs, [True] * len(many), hay=hay)
        assert passes(rs) == 2
        close_all(rs)
        rs, _ = hs.search_hamming_batch(dup, dup_k)
        check(hs, dup, dup_k, rs, [True] * len(dup))
        assert passes(rs) == 1 and all(r.count(F.RAW) >= 2 for r in rs)
        close_all(rs)
        tiny_pats, tiny_k = many[:10], many_k[:10]  # more than 8 records in the pass
        rs, _ = hs.search_hamming_batch(tiny_pats, tiny_k, F.F_TINY_LIST)
        check(hs, tiny_pats, tiny_k, rs, [False] * len(tiny_pats), hay=hay)
        assert sum(r.count(F.RAW) for r in rs) > 8
        close_all(rs)
        rs, _ = hs.search_hamming_batch(tiny_pats, tiny_k)
        check(hs, tiny_pats, tiny_k, rs, [True] * len(tiny_pats), hay=hay)
        close_all(rs)
    hs.close()


LIMITS = [  # one pattern of each search class, and one more substitutions-only
    dict(max_l_dist=0),                                              # ExactSearch
    dict(max_substitutions=2, max_insertions=0, max_deletions=0),    # SubstitutionsOnlySearch
    dict(max_l_dist=2),                                              # LevenshteinSearch
    dict(max_substitutions=1, max_insertions=1, max_deletions=0, max_l_dist=2),  # GenericSearch
    dict(max_substitutions=3, max_insertions=0, max_deletions=0, max_l_dist=1),  # substitutions-only, 1 effective
]


def per_pattern_limits(limits):
    keys = ("max_substitutions", "max_insertions", "max_deletions", "max_l_dist")
    return {key: [d.get(key) for d in limits] for key in keys}


def sequences(rng):
    """the same text as every sequence kind the package takes -> [(sequence, patterns)]"""
    base = rand_bytes(rng, b"ACGTN", 6000)
    pats = [base[100:112], base[2000:2024], base[3000:3020], base[4000:4018], base[5000:5030]]
    pats = [substitute(rng, p, b"ACGT", 1) for p in pats]
    wide = base.decode("latin-1").translate(str.maketrans("ACGTN", "αβγδε"))
    wpats = [p.decode("latin-1").translate(str.maketrans("ACGTN", "αβγδε")) for p in pats]
    return [(base, pats), (bytearray(base), [bytearray(p) for p in pats]), (base.decode("latin-1"),
            [p.decode("latin-1") for p in pats]), (wide, wpats), (list(base), [list(p) for p in pats]),
            (DeviceSequence(base), pats)]


def test_public_api_mixes_every_search_class(cuda_device):
    """find_near_matches_batch with per-pattern limits of all four search classes equals find_near_matches per
    pattern (Match.matched included) for bytes, bytearray, str (latin-1 and wide), list and DeviceSequence; invalid
    limits raise what find_near_matches raises."""
    rng = np.random.default_rng(8106)
    lim = per_pattern_limits(LIMITS)
    for seq, pats in sequences(rng):
        got = find_near_matches_batch(pats, seq, **lim)
        want = [find_near_matches(p, seq, **d) for p, d in zip(pats, LIMITS)]
        assert got == want, type(seq)
        assert all(len(w) for w in want[1:])
        # one int for a limit applies to every pattern
        assert find_near_matches_batch(pats, seq, max_substitutions=2, max_insertions=0, max_deletions=0) == \
            [find_near_matches(p, seq, max_substitutions=2, max_insertions=0, max_deletions=0) for p in pats]
    seq, pats = sequences(rng)[0]
    for bad in (dict(max_substitutions=-1, max_insertions=0, max_deletions=0), dict(max_substitutions=2),
                dict(max_substitutions=1, max_deletions=0), dict(), dict(max_l_dist=1.5)):
        with pytest.raises(Exception) as single:
            find_near_matches(pats[0], seq, **bad)
        with pytest.raises(Exception) as batch:
            find_near_matches_batch(pats, seq, **bad)
        assert type(batch.value) is type(single.value) and str(batch.value) == str(single.value), bad
    for kw in (dict(max_l_dist=0), dict(max_substitutions=1, max_insertions=0, max_deletions=0), dict(max_l_dist=1)):
        with pytest.raises(ValueError) as single:
            find_near_matches(b"", seq, **kw)
        with pytest.raises(ValueError) as batch:
            find_near_matches_batch([pats[0], b""], seq, **kw)
        assert str(batch.value) == str(single.value)
    with pytest.raises(ValueError):
        find_near_matches_batch(pats, seq, max_l_dist=[1, 2])


def test_dna_workload_at_4_gib(cuda_device):
    """The probe's DNA workload (tools/probe_ham_batch.py) on 4 GiB: every list equals its single search."""
    needs_real_gpu("4 GiB haystack")
    sys.path.insert(0, os.path.join(os.path.dirname(os.path.dirname(os.path.abspath(__file__))), "tools"))
    import probe_ham_batch
    hs, pats, ks = probe_ham_batch.make_haystack("dna", 4 << 30)
    rs, _ = hs.search_hamming_batch(pats, ks)
    routes = [r.stats()["route"] for r in rs]
    assert routes.count(SHARED) >= len(pats) // 2
    for p, k, r in zip(pats, ks, rs):
        one = hs.search_hamming(p, k)
        assert probe_ham_batch.same(probe_ham_batch.lists(r), probe_ham_batch.lists(one)), (p, k)
        assert r.count(F.RAW) >= 1
        one.close()
        r.close()
    hs.close()
