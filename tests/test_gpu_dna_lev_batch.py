"""Levenshtein batches on low-entropy sequences (DNA): the n-gram-route patterns no other shared pass takes share 2-bit
n-gram scans (k_filter_mdense2 -> k_verify_mhits, DESIGN.md section 5.12).  Every case checks, pattern by pattern,
that the batch's RAW list with anchors (in order), FINAL list and group rows equal the single search_levenshtein on
the same handle, and the oracle where the size allows, and which patterns rode on a shared scan (a shared pass
reports its scan on its first pattern only; the others report no bytes).  `small` keeps the sizes the CPU emulator
replays (tests/test_emu_dna_lev_batch.py)."""
import numpy as np
import pytest

import oracle
from conftest import needs_real_gpu
from corpus import ASCII, DNA, mutate
from fuzzysearch_b200 import DeviceSequenceSet, _native as F, find_near_matches, find_near_matches_batch, \
    find_near_matches_batch_in_each
from parity import tup
from test_gpu_records import rand
from test_gpu_records_batch import _each, check_batch

pytestmark = pytest.mark.gpu

DENSE = "ngrams/dense-filter"
TINY_CHUNK = 3000  # FZB_F_TINY_LIST: positions per chunk of the 2-bit pass


def rows(res):
    s, e, d, ng, ix = res.arrays(F.RAW, anchors=True)
    return list(zip(s.tolist(), e.tolist(), d.tolist(), ng.tolist(), ix.tolist()))


def same(a, b):
    """RAW with anchors (in order), FINAL and group rows of two results are equal"""
    return (all(np.array_equal(x, y) for x, y in zip(a.arrays(F.RAW, anchors=True), b.arrays(F.RAW, anchors=True)))
            and all(np.array_equal(x, y) for x, y in zip(a.arrays(F.FINAL), b.arrays(F.FINAL)))
            and np.array_equal(a.group_rows(), b.group_rows()))


def riders(results):
    """patterns that rode on another pattern's 2-bit scan"""
    return [q for q, r in enumerate(results) if r.stats()["route"] == DENSE and r.stats()["bytes_scanned"] == 0]


def check(hs, pats, ks, results, hay=None):
    """each result equals the single search on `hs`; with `hay` (the whole sequence) also the oracle"""
    assert len(results) == len(pats)
    for q, (p, k, r) in enumerate(zip(pats, ks, results)):
        one = hs.search_levenshtein(p, k)
        ctx = (q, len(p), k)
        route = one.stats()["route"]
        assert r.stats()["route"] == route, ctx
        assert same(r, one), ctx
        one.close()
        if hay is not None:
            raw = oracle.levenshtein_raw(p, bytes(hay), k)
            got = r.triples(F.RAW)
            assert (sorted(got) == sorted(tup(raw))) if route == "exact" else (got == tup(raw)), ctx
            if k:
                assert r.triples(F.FINAL) == tup(oracle.consolidate(raw)), ctx


def close_all(results):
    for r in results:
        r.close()


def dna_hay(rng, n, n_runs=6):
    hay = np.frombuffer(rand(rng, DNA, n), dtype=np.uint8).copy()
    for _ in range(n_runs):  # runs of N and of another letter: both alias to some code of the 2-bit keys
        pos = int(rng.integers(0, n - 100))
        hay[pos:pos + int(rng.integers(10, 90))] = ord("N" if rng.random() < 0.5 else "R")
    return hay


def plant(rng, hay, pat, k, pos):
    v = mutate(rng, pat, DNA, int(rng.integers(0, k + 1)))[:len(hay) - pos]
    hay[pos:pos + len(v)] = np.frombuffer(v, dtype=np.uint8)


def shape_mix(rng):
    """-> (patterns, ks, shared?): n-grams of 5, 6, 7 (keys with completions), 8 and more symbols; duplicates, a prefix
    of another pattern, periodic patterns with repeated n-grams, non-ACGT bytes; and patterns the pass leaves alone"""
    pats, ks, shared = [], [], []

    def add(p, k, s):
        pats.append(p)
        ks.append(k)
        shared.append(s)

    for m, k in ((15, 2), (11, 1), (18, 2), (13, 1), (14, 1), (21, 2), (16, 1), (24, 2), (20, 1), (33, 2), (40, 1),
                 (64, 1), (40, 2)):
        add(rand(rng, DNA, m), k, True)
    add(pats[0], 2, True)                        # a duplicate
    add(pats[2], 1, True)                        # the same bytes with another k
    add(pats[9][:17], 2, True)                   # a prefix of another pattern (L = 5)
    add(b"ACGTAC" * 3, 2, True)                  # three equal n-grams
    add(b"A" * 20, 3, True)                      # periodic, L = 5
    add(rand(rng, DNA, 9) + b"N" + rand(rng, DNA, 10), 1, True)  # a byte outside the four codes
    add(b"RR" + rand(rng, DNA, 16), 2, True)
    add(rand(rng, DNA, 12), 2, False)            # L = 4: too short for the key
    add(rand(rng, DNA, 9), 1, False)             # L = 4
    add(rand(rng, DNA, 70), 2, False)            # m > 64
    add(rand(rng, DNA, 40), 0, False)            # exact
    add(rand(rng, DNA, 60), 2, False)            # m - L > 32
    return pats, ks, shared


def test_key_lengths_and_pattern_shapes(cuda_device, small=False):
    rng = np.random.default_rng(5120)
    n = 20000 if small else 200000
    pats, ks, shared = shape_mix(rng)
    hay = dna_hay(rng, n)
    for p, k in zip(pats, ks):
        for _ in range(3):
            plant(rng, hay, p, k, int(rng.integers(0, n - len(p))))
    hay[:len(pats[1])] = np.frombuffer(pats[1], dtype=np.uint8)        # a match at 0
    hay[n - len(pats[7]):] = np.frombuffer(pats[7], dtype=np.uint8)    # and at N - m
    hs = F.Haystack.from_host(hay)
    for _ in range(2):  # twice on the same handle
        res, total = hs.search_levenshtein_batch(pats, ks)
        got = riders(res)
        assert set(got) | {min(q for q, s in enumerate(shared) if s)} == {q for q, s in enumerate(shared) if s}, got
        assert len(got) == sum(shared) - 1  # one pass
        assert total["route"] == "batch"
        check(hs, pats, ks, res, hay=hay)
        assert (0, len(pats[1]), 0) in res[1].triples(F.FINAL)
        assert (n - len(pats[7]), n, 0) in res[7].triples(F.FINAL)
        close_all(res)
    hs.close()


def test_tile_packed_with_occurrences(cuda_device, small=False):
    """More hits in one 64 KiB tile than a CTA buffers (3 072; flushed at 1 024): flushes and spills to the list"""
    rng = np.random.default_rng(5121)
    n = 40000 if small else 1 << 18
    pats = [rand(rng, DNA, 15), rand(rng, DNA, 20)]
    ks = [2, 1]
    hay = dna_hay(rng, n)
    copies = 700 if small else 1100  # (either way more than 3 072 hits in the tile)
    run = (pats[0] * copies + pats[1] * copies)[:n - 5000]
    hay[1000:1000 + len(run)] = np.frombuffer(run, dtype=np.uint8)
    hs = F.Haystack.from_host(hay)
    res, _ = hs.search_levenshtein_batch(pats, ks)
    assert riders(res) == [1]
    assert res[0].stats()["n_candidates"] >= 3 * copies + 2 * copies
    check(hs, pats, ks, res, hay=hay)
    close_all(res)
    hs.close()


def test_tiny_lists_chunk_seams_and_overflow(cuda_device, small=False):
    """FZB_F_TINY_LIST: chunks of 3 000 positions with a hit list of 8.  Occurrences straddle every seam (their
    n-grams on either side); then more than 8 hits in one chunk send every pattern one by one."""
    rng = np.random.default_rng(5122)
    n = 7 * TINY_CHUNK + 123
    pats = [rand(rng, DNA, m) for m in (20, 24, 30, 40)]  # two n-grams of 10 symbols and more: no random hits
    ks = [1, 1, 1, 1]
    hay = dna_hay(rng, n, n_runs=0)
    firsts = []
    for c in range(1, 7):  # at most 6 hits per chunk
        seam = c * TINY_CHUNK
        p = pats[c % 4]
        # the last start of a chunk, the first start of the next, or n-grams on both sides of the seam
        first = seam - 1 if c % 2 else seam if c == 6 else seam - len(p) // 2
        firsts.append(first)
        for pos, q in ((first, p), (seam - 100, pats[(c + 1) % 4])):
            hay[pos:pos + len(q)] = np.frombuffer(q, dtype=np.uint8)
    hs = F.Haystack.from_host(hay)
    res, total = hs.search_levenshtein_batch(pats, ks, F.F_TINY_LIST)
    assert riders(res) == [1, 2, 3]
    assert res[0].stats()["n_launches"] == 2 * ((n + TINY_CHUNK - 1) // TINY_CHUNK)  # scan + verify per chunk
    check(hs, pats, ks, res, hay=hay)
    starts = {s for r in res for s, _, _ in r.triples(F.FINAL)}
    assert all(f in starts for f in firsts) and all(c * TINY_CHUNK - 100 in starts for c in range(1, 7))
    normal, _ = hs.search_levenshtein_batch(pats, ks)
    for a, b in zip(res, normal):
        assert same(a, b)
    close_all(res)
    close_all(normal)
    hs.close()
    run = pats[0] * 12  # 12 occurrences (24 hits) inside one chunk
    hay[5000:5000 + len(run)] = np.frombuffer(run, dtype=np.uint8)
    hs = F.Haystack.from_host(hay)
    res, _ = hs.search_levenshtein_batch(pats, ks, F.F_TINY_LIST)
    assert all(r.stats()["bytes_scanned"] == n for r in res)  # every pattern on its own
    check(hs, pats, ks, res, hay=hay)
    close_all(res)
    hs.close()


def test_at_64_bit_offsets(cuda_device, small=False):
    """The same bytes as an interior shard at global offsets up to 2^44: the batch at each offset is the batch at
    offset 0, shifted (the hit list packs buffer-relative positions into 40 bits)."""
    rng = np.random.default_rng(5123)
    n = 20000 if small else 100000
    pats = [rand(rng, DNA, m) for m in (15, 18, 24, 40)]
    ks = [2, 2, 1, 1]
    hay = dna_hay(rng, n)
    for p, k in zip(pats, ks):
        for _ in range(4):
            plant(rng, hay, p, k, int(rng.integers(300, n - 400)))
    lo, hi = 256, n - 256
    a = F.Haystack.from_host(hay, buf_lo=0, global_len=n + (1 << 20), own_lo=lo, own_hi=hi)
    ra, _ = a.search_levenshtein_batch(pats, ks)
    assert riders(ra) == [1, 2, 3]
    check(a, pats, ks, ra)
    for shift in (1 << 32, (1 << 40) + 16 * 12345, 1 << 44):
        b = F.Haystack.from_host(hay, buf_lo=shift, global_len=shift + n + (1 << 20), own_lo=shift + lo,
                                 own_hi=shift + hi)
        rb, _ = b.search_levenshtein_batch(pats, ks)
        assert riders(rb) == [1, 2, 3]
        for x, y in zip(ra, rb):
            assert [(s + shift, e + shift, d, g, i + shift) for s, e, d, g, i in rows(x)] == rows(y), hex(shift)
            assert [(s + shift, e + shift, d) for s, e, d in x.triples(F.FINAL)] == y.triples(F.FINAL), hex(shift)
        close_all(rb)
        b.close()
    close_all(ra)
    a.close()


def test_records_and_public_api(cuda_device, small=False):
    """FZB_F_PER_RECORD on a set of reads (record edges, occurrences across separators), the public batch functions on
    bytes, a resident set and a general-Unicode DNA str (reduced to bytes 1..4 on the device)"""
    rng = np.random.default_rng(5124)
    pats = [rand(rng, DNA, m) for m in (15, 16, 20, 24, 18)]
    ks = [2, 1, 1, 2, 1]
    nrec = 60 if small else 2000
    recs = [bytearray(rand(rng, DNA, int(x))) for x in rng.integers(0, 200, size=nrec)]
    for i, r in enumerate(recs[:-1]):
        p = pats[i % len(pats)]
        if len(r) >= len(p) and len(recs[i + 1]) >= len(p):
            if i % 3 == 0:  # across the separator
                cut = int(rng.integers(1, len(p)))
                r[len(r) - cut:] = p[:cut]
                recs[i + 1][:len(p) - cut] = p[cut:]
            elif i % 3 == 1:  # at the record's end
                r[len(r) - len(p):] = mutate(rng, p, DNA, 1)[:len(p)]
            else:
                r[:len(p)] = p
    recs = [bytes(r) for r in recs]
    check_batch(recs, "lev", pats, ks, shared=(DENSE,))
    check_batch(recs, "lev", pats, ks, F.F_TINY_LIST, with_oracle=False)
    for lim in (dict(max_l_dist=1), dict(max_l_dist=ks)):
        want = _each(pats, recs, lim)
        assert find_near_matches_batch_in_each(pats, recs, **lim) == want
        resident = DeviceSequenceSet(recs)
        assert find_near_matches_batch_in_each(pats, resident, **lim) == want
        resident.close()
    hay = "".join(r.decode() for r in recs[:40]) + "αω" + "".join(r.decode() for r in recs[40:])
    tp = [p.decode() for p in pats]
    assert find_near_matches_batch(tp, hay, max_l_dist=1) == [find_near_matches(p, hay, max_l_dist=1) for p in tp]
    # what the device reduction makes of that str: the pattern symbols as bytes 1..4, the others as 5; the pass runs
    # on it (its code table comes from the pass's pattern bytes, not from the letters ACGT)
    code = bytes.maketrans(b"ACGT", b"\1\2\3\4")
    red = np.frombuffer(hay.encode("utf-8").replace("αω".encode("utf-8"), b"\5\5").translate(code), dtype=np.uint8)
    rpats = [p.translate(code) for p in pats]
    hs = F.Haystack.from_host(red)
    res, _ = hs.search_levenshtein_batch(rpats, [1] * len(rpats))
    assert riders(res) == list(range(1, len(rpats)))
    check(hs, rpats, [1] * len(rpats), res, hay=red)
    close_all(res)
    hs.close()


def test_patterns_left_one_by_one(cuda_device, small=False):
    """Other flags, a sequence just below the 0.15 collision probability and an ASCII sequence: the 2-bit pass does not
    run, and the lists still equal the single searches"""
    rng = np.random.default_rng(5125)
    n = 20000 if small else 100000
    pats = [rand(rng, DNA, m) for m in (15, 20, 24)]
    ks = [2, 1, 2]
    hay = dna_hay(rng, n)
    for p, k in zip(pats, ks):
        plant(rng, hay, p, k, int(rng.integers(0, n - len(p))))
    hs = F.Haystack.from_host(hay)
    for flags in (F.F_NO_FINAL, F.F_FORCE_DENSE):
        res, _ = hs.search_levenshtein_batch(pats, ks, flags)
        assert all(r.stats()["bytes_scanned"] == n for r in res), flags
        for p, k, r in zip(pats, ks, res):
            one = hs.search_levenshtein(p, k, flags)
            assert rows(r) == rows(one), flags
            one.close()
        close_all(res)
    hs.close()
    # 7 letters (c = 1/7): the prefix pass takes three patterns with two n-grams each (0.0175 expected prefix hits per
    # position; a fourth would pass 0.02), the 2-bit pass none of the other three, which it would take at c >= 0.15
    seven = np.frombuffer(rand(rng, b"ACGTNRY", n), dtype=np.uint8).copy()
    spats = [rand(rng, b"ACGTNRY", 11) for _ in range(6)]
    for p in spats:
        plant(rng, seven, p, 1, int(rng.integers(0, n - len(p))))
    hs = F.Haystack.from_host(seven)
    res, _ = hs.search_levenshtein_batch(spats, [1] * 6)
    assert riders(res) == [1, 2]
    assert [r.stats()["bytes_scanned"] for r in res] == [n, 0, 0, n, n, n]
    check(hs, spats, [1] * 6, res, hay=seven)
    close_all(res)
    hs.close()
    text = np.frombuffer(rand(rng, ASCII, n), dtype=np.uint8).copy()
    tpats = [rand(rng, ASCII, m) for m in (15, 20, 24)]
    for p, k in zip(tpats, ks):
        plant_text = mutate(rng, p, ASCII, k)
        pos = int(rng.integers(0, n - len(plant_text)))
        text[pos:pos + len(plant_text)] = np.frombuffer(plant_text, dtype=np.uint8)
    hs = F.Haystack.from_host(text)
    res, _ = hs.search_levenshtein_batch(tpats, ks)
    assert riders(res) == []  # two patterns share the q-sample pass, one goes alone
    check(hs, tpats, ks, res, hay=text)
    close_all(res)
    hs.close()


def test_full_size(cuda_device):
    """4 GiB of DNA and 1 024 patterns (m 15-40, k 1-2) with plants: every pattern with n-grams of 6 symbols or more
    rides on one 2-bit scan, those with n-grams of 5 (m 15-17, k 2), which cost more in the pass than alone on 4 GiB,
    go one by one; every list equals its single search"""
    needs_real_gpu("4 GiB input")
    rng = np.random.default_rng(5126)
    n = 4 << 30
    hs = F.Haystack.alloc(n)
    hs.fill_synthetic(DNA, 29)
    pats, ks = [], []
    for _ in range(1024):
        m = int(rng.integers(15, 41))
        pats.append(rand(rng, DNA, m))
        ks.append(int(rng.integers(1, 3)))
    for p, k in zip(pats, ks):
        for _ in range(4):
            hs.write(int(rng.integers(0, n - 64)), mutate(rng, p, DNA, int(rng.integers(0, k + 1))))
    res, total = hs.search_levenshtein_batch(pats, ks)
    alone = [q for q, (p, k) in enumerate(zip(pats, ks)) if len(p) // (k + 1) == 5]
    ride = set(riders(res))
    assert 40 <= len(alone) and not ride & set(alone)
    assert len(ride) == len(pats) - len(alone) - 1  # one pass: its first pattern reports the scan
    assert sum(r.count(F.RAW) for r in res) >= 4 * len(pats)
    for q, (p, k, r) in enumerate(zip(pats, ks, res)):
        one = hs.search_levenshtein(p, k)
        assert same(r, one), q
        one.close()
    close_all(res)
    hs.close()
