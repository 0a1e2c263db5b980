"""GPU vs CPU oracle on seeded corpora with planted near-matches (sizes the oracle handles in
seconds), incl. sharded searches whose union must equal the single-shard raw stream."""
import numpy as np
import pytest

import oracle
from corpus import ASCII, DNA, make_corpus
from fuzzysearch_b200 import _native as F
from parity import tup

pytestmark = pytest.mark.gpu


def _raw(res):
    s, e, d, ng, ix = res.arrays(F.RAW, anchors=True)
    return list(zip(s.tolist(), e.tolist(), d.tolist())), ng.tolist(), ix.tolist()


@pytest.mark.parametrize("alphabet,n,m,k,flags", [
    (ASCII, 1 << 22, 20, 2, 0),
    (ASCII, 1 << 22, 20, 2, F.F_FORCE_DENSE),
    (ASCII, 1 << 22, 20, 2, F.F_TINY_LIST),   # granule work list overflows -> bitmap sweep
    (DNA, 1 << 18, 20, 2, F.F_TINY_LIST | F.F_FORCE_SAMPLED),
    (DNA, 1 << 20, 20, 2, F.F_FORCE_SAMPLED),  # non-selective sampled filter: nearly every granule marked
    (DNA, 1 << 16, 30, 3, 0),                  # L = 7: dense filter hashes 7-byte n-grams
    (DNA, 1 << 18, 20, 2, F.F_TINY_LIST),      # hit list overflows -> retry in granule mode (tiny work list)
    (b"ab", 1 << 14, 50, 4, 0),                # L = 10 > 8: dense filter on an 8-byte prefix
    (ASCII, (1 << 20) + 13, 32, 3, 0),
    (ASCII, 1 << 20, 9, 2, 0),          # L = 3: dense filter, q = 3
    (ASCII, 1 << 20, 64, 4, 0),
    (DNA, 1 << 20, 20, 2, 0),           # config 1 of BASELINE.json
    (DNA, 1 << 18, 20, 2, F.F_FORCE_DENSE),
    (DNA, 1 << 18, 12, 1, 0),
    (b"ab", 1 << 14, 12, 2, 0),
])
def test_levenshtein_ngrams_matches_oracle(cuda_device, alphabet, n, m, k, flags):
    pat, hay, _ = make_corpus(11, n, alphabet, m, 64, k + 1)
    raw_cpu, ng_cpu, ix_cpu = oracle.levenshtein_ngrams_raw(pat, hay, k, with_anchor=True)
    hs = F.Haystack.from_host(hay)
    res = hs.search_levenshtein(pat, k, flags)
    raw_gpu, ng, ix = _raw(res)
    assert raw_gpu == tup(raw_cpu)
    assert ng == ng_cpu.tolist() and ix == ix_cpu.tolist()
    assert res.triples(F.FINAL) == tup(oracle.consolidate(raw_cpu))
    assert len(raw_gpu) >= 32
    res.close()
    hs.close()


@pytest.mark.parametrize("alphabet,n,m,k,flags", [
    (DNA, 1 << 20, 32, 3, 0),   # config 3 of BASELINE.json (scaled): counting filter (TMA tiles)
    (DNA, (1 << 20) + 77, 32, 3, 0),
    (DNA, 1 << 18, 32, 3, F.F_FORCE_DENSE),   # brute-force fallback kernel
    (ASCII, 1 << 20, 32, 3, 0),
    (b"ab", 1 << 16, 40, 5, 0),  # tiny alphabet, repeated grams, Wc = 8 < W
    (b"ab", 1 << 14, 64, 7, 0),
    (DNA, 300, 32, 3, 0),        # shorter than one tile
    (DNA, 1 << 16, 11, 1, 0),    # smallest m for k = 1 (W = 2)
    (DNA, 1 << 16, 8, 2, 0),     # lemma does not apply -> fallback
    (b"ab", 1 << 12, 6, 5, 0),
    (ASCII, 1 << 12, 5, 7, 0),   # k >= m: every start matches
])
def test_hamming_matches_oracle(cuda_device, alphabet, n, m, k, flags):
    pat, hay, _ = make_corpus(5, n, alphabet, m, 64, k + 1, subs_only=True)
    cpu = oracle.substitutions(pat, hay, k)
    hs = F.Haystack.from_host(hay)
    res = hs.search_hamming(pat, k, flags)
    assert res.triples(F.RAW) == tup(cpu)
    assert res.triples(F.FINAL) == tup(cpu)
    res.close()
    hs.close()


@pytest.mark.parametrize("alphabet,n,m,k", [
    (ASCII, 1 << 18, 8, 2),
    (DNA, 1 << 14, 8, 2),
    (DNA, 1 << 12, 5, 3),
    (b"ab", 1 << 9, 4, 2),
    (ASCII, 1 << 10, 3, 4),  # k >= m
])
def test_levenshtein_lp_matches_oracle(cuda_device, alphabet, n, m, k):
    pat, hay, _ = make_corpus(3, n, alphabet, m, 32, k + 1)
    cpu = oracle.levenshtein_lp_raw(pat, hay, k)
    hs = F.Haystack.from_host(hay)
    res = hs.search_levenshtein(pat, k, F.F_FORCE_LP)
    assert sorted(res.triples(F.RAW)) == sorted(tup(cpu))
    assert res.triples(F.FINAL) == tup(oracle.consolidate(cpu))
    res.close()
    hs.close()


@pytest.mark.parametrize("alphabet,n,m,limits,flags", [
    (ASCII, 1 << 18, 20, (2, 1, 1, 3), 0),
    (ASCII, 1 << 16, 20, (2, 1, 1, 3), F.F_FORCE_DENSE),
    (DNA, 1 << 13, 20, (2, 1, 1, 3), 0),
    (DNA, 1 << 12, 12, (1, 1, 0, 2), 0),
    (ASCII, 1 << 14, 8, (1, 2, 1, 3), F.F_FORCE_LP),
    (DNA, 1 << 11, 6, (2, 0, 2, 3), F.F_FORCE_LP),
    # limits far above what 20 symbols can spend (max_l_dist=None -> the sum, common.py:86-104): the LP route lowers
    # the total to m + max_insertions, which cannot change the raw stream (search_generic, api.cu)
    (ASCII, 1 << 12, 20, (100, 1, 1, 102), F.F_FORCE_LP),
    (b"abcd", 1 << 9, 12, (50, 2, 50, 102), F.F_FORCE_LP),
])
def test_generic_matches_oracle(cuda_device, alphabet, n, m, limits, flags):
    pat, hay, _ = make_corpus(9, n, alphabet, m, 32, limits[3] + 1)
    if flags & F.F_FORCE_LP:
        cpu = oracle.generic_lp_raw(pat, hay, *limits)
    else:
        cpu = oracle.generic_ngrams_raw(pat, hay, *limits)
    hs = F.Haystack.from_host(hay)
    res = hs.search_generic(pat, *limits, flags=flags)
    assert sorted(res.triples(F.RAW)) == sorted(tup(cpu))
    assert res.triples(F.FINAL) == tup(oracle.consolidate(cpu))
    res.close()
    hs.close()


@pytest.mark.parametrize("nshards", [2, 3, 7])
def test_sharded_union_equals_whole(cuda_device, nshards):
    """SURVEY 8e: shards own anchors in [lo,hi) and carry a halo of m+k; the union of the shards'
    raw streams is the single-device raw stream (matches straddling every seam are planted)."""
    m, k, n = 20, 2, (1 << 20) + 5
    pat, hay, _ = make_corpus(21, n, ASCII, m, 64, 3)
    bounds = [((n * i // nshards) // 16) * 16 for i in range(nshards)] + [n]
    for b in bounds[1:-1]:  # straddle every seam at the deltas of test_find_near_matches_in_file.py:84-86
        for j, delta in enumerate((-m, -m + 1, -4, -2, -1, 0, 1)):
            pos = b + delta + 64 * (j - 3)
            hay[pos:pos + m] = np.frombuffer(pat, dtype=np.uint8)
        hay[b - 7:b - 7 + m] = np.frombuffer(pat, dtype=np.uint8)
    whole = tup(oracle.levenshtein_ngrams_raw(pat, hay, k))
    halo = m + k
    got = []
    for i in range(nshards):
        lo, hi = bounds[i], bounds[i + 1]
        blo = max(0, lo - halo) // 16 * 16
        bhi = min(n, hi + halo)
        hs = F.Haystack.from_host(hay[blo:bhi], buf_lo=blo, global_len=n, own_lo=lo, own_hi=hi)
        res = hs.search_levenshtein(pat, k, F.F_NO_FINAL)
        s, e, d, ng, ix = res.arrays(F.RAW, anchors=True)
        got += list(zip(ng.tolist(), ix.tolist(), s.tolist(), e.tolist(), d.tolist()))
        res.close()
        hs.close()
    got.sort()
    assert [(s, e, d) for _, _, s, e, d in got] == whole
    hs = F.Haystack.from_host(hay)
    ham_whole = hs.search_hamming(pat, 3).triples(F.RAW)
    hs.close()
    ham = []
    for i in range(nshards):
        lo, hi = bounds[i], bounds[i + 1]
        blo = max(0, lo - halo) // 16 * 16
        bhi = min(n, hi + halo)
        hs = F.Haystack.from_host(hay[blo:bhi], buf_lo=blo, global_len=n, own_lo=lo, own_hi=hi)
        ham += hs.search_hamming(pat, 3).triples(F.RAW)
        hs.close()
    assert sorted(ham) == ham_whole


def test_edge_cases(cuda_device):
    from fuzzysearch_b200 import find_near_matches
    t = lambda ms: [(m.start, m.end, m.dist) for m in ms]  # noqa: E731
    assert t(find_near_matches(b"abc", b"", max_l_dist=1)) == []
    assert t(find_near_matches(b"ab", b"xyz", max_l_dist=2)) == [(0, 0, 2), (1, 1, 2), (2, 2, 2), (3, 3, 2)]
    assert t(find_near_matches(b"ab", b"xyz", max_l_dist=10 ** 6)) == [(0, 0, 2), (1, 1, 2), (2, 2, 2), (3, 3, 2)]
    assert t(find_near_matches(b"abc", b"ab", max_l_dist=1)) == [(0, 2, 1)]
    assert t(find_near_matches(b"abc", b"xbz", max_substitutions=5, max_insertions=0, max_deletions=0)) == \
        [(0, 3, 2)]
    assert t(find_near_matches(b"abcd", b"ab", max_substitutions=1, max_insertions=0, max_deletions=0)) == []
    from fuzzysearch_b200 import has_near_match
    assert has_near_match(b"PATTERN", b"---PATERN---", max_l_dist=1) is True
    assert has_near_match(b"PATTERN", b"---PATERN---", max_l_dist=0) is False
    assert has_near_match(b"abc", b"xbz", max_substitutions=1, max_insertions=0, max_deletions=0) is False
    ms = find_near_matches(b"PATTERN", b"---PATERN---", max_l_dist=1)
    assert t(ms) == [(3, 9, 1)] and ms[0].matched == b"PATERN"
    ms = find_near_matches("PATTERN", "---PATERN---", max_l_dist=1)
    assert ms[0].matched == "PATERN"
    with pytest.raises(ValueError):
        find_near_matches(b"", b"TEXT", max_l_dist=1)
    with pytest.raises(ValueError):
        find_near_matches(b"a", b"a")
    with pytest.raises(TypeError):
        find_near_matches(b"a", b"a", max_l_dist=-1)
    # item sequences (tests/test_gpu_symbols.py); max_l_dist >= len(subsequence): the LP route's empty match at
    # every index (levenshtein.py:62-65) -- what the reference returns for these very inputs
    assert t(find_near_matches(["a"], ["a"], max_l_dist=1)) == [(0, 0, 1), (1, 1, 1)]
    assert t(find_near_matches(["a", "b"], ["a", "b", "c"], max_l_dist=1)) == [(0, 2, 0)]
    with pytest.raises(TypeError):
        find_near_matches(["a"], b"a", max_l_dist=1)


def test_python_surface_variants(cuda_device):
    """bytes / bytearray / memoryview / numpy / latin-1 str / DeviceSequence all take the same path."""
    from fuzzysearch_b200 import DeviceSequence, Match, find_near_matches
    pat, hay, _ = make_corpus(8, 1 << 16, ASCII, 12, 16, 2)
    exp = oracle.find_near_matches(pat, hay, max_l_dist=1)
    raw = hay.tobytes()
    for seq in (raw, bytearray(raw), memoryview(raw), hay, raw.decode("latin-1")):
        p = pat.decode("latin-1") if isinstance(seq, str) else pat
        ms = find_near_matches(p, seq, max_l_dist=1)
        assert [(m.start, m.end, m.dist) for m in ms] == exp
        assert all(isinstance(m, Match) for m in ms)
        want = seq[ms[0].start:ms[0].end]
        assert ms[0].matched == (bytes(want) if not isinstance(seq, str) else want)
    dev = DeviceSequence(raw)
    for k in (0, 1, 2):
        ms = find_near_matches(pat, dev, max_l_dist=k)
        assert [(m.start, m.end, m.dist) for m in ms] == oracle.find_near_matches(pat, hay, max_l_dist=k)
    ms = find_near_matches(pat, dev, max_substitutions=2, max_insertions=0, max_deletions=0)
    assert [(m.start, m.end, m.dist) for m in ms] == oracle.find_near_matches(pat, hay, 2, 0, 0)
    assert len(dev) == len(raw)
    dev.close()
    with pytest.raises(TypeError):
        find_near_matches(pat, raw.decode("latin-1"), max_l_dist=1)   # bytes pattern vs str sequence


def test_positions_are_64_bit_everywhere(cuda_device):
    """A shard far inside a huge global sequence (offsets up to 2^44) must report what the same bytes report at
    offset 0, shifted: every route, raw and final, also through the work-list overflow path.  (BASELINE configs[3]
    reaches 2^35; the full-size bench checks that one offset, this checks the arithmetic.)"""
    rng = np.random.default_rng(4)
    for trial in range(12):
        alphabet = [ASCII, DNA, b"abcdefgh"][trial % 3]
        m = int(rng.choice([5, 8, 12, 20, 33, 64, 100]))
        k = int(rng.integers(0, min(m // 3, 4) + 1))
        n = 4096 if len(alphabet) <= 4 else int(rng.choice([4096, 70000]))
        pat, hay, _ = make_corpus(100 + trial, n, alphabet, m, 10, k + 1, clusters=2)
        shift = int(rng.choice([1 << 32, (1 << 35) - 4096, (1 << 40) + 16 * 12345, 1 << 44]))
        lo, hi = 256, n - 256  # interior anchors, halo on both sides, no global end in sight
        a = F.Haystack.from_host(hay, buf_lo=0, global_len=n + (1 << 20), own_lo=lo, own_hi=hi)
        b = F.Haystack.from_host(hay, buf_lo=shift, global_len=shift + n + (1 << 20), own_lo=shift + lo,
                                 own_hi=shift + hi)
        calls = [lambda h: h.search_levenshtein(pat, k), lambda h: h.search_hamming(pat, min(k, 3)),
                 lambda h: h.search_exact(pat), lambda h: h.search_levenshtein(pat, k, F.F_FORCE_DENSE),
                 lambda h: h.search_levenshtein(pat, k, F.F_TINY_LIST)]
        if k >= 1:
            calls.append(lambda h: h.search_generic(pat, k, 1, 1, k))
        for ci, call in enumerate(calls):
            ra, rb = call(a), call(b)
            for which in (F.RAW, F.FINAL):
                ta, tb = sorted(ra.triples(which)), sorted(rb.triples(which))
                assert [(s + shift, e + shift, d) for s, e, d in ta] == tb, (trial, ci, which, m, k, hex(shift))
            ra.close()
            rb.close()
        a.close()
        b.close()
    # the last positions a handle can hold: k_post's keys and k_merge's scores keep a position in 46 bits, so a shard
    # may end at global_len = 2^46 - 1 (the LP route's empty match (N, N, m) included) and no further
    top = (1 << 46) - 1
    n = 4095  # the shard's buf_lo = top - n is a multiple of 16
    pat, hay, _ = make_corpus(46, n, ASCII, 20, 10, 3)
    a = F.Haystack.from_host(hay, buf_lo=0, global_len=n, own_lo=256, own_hi=n)
    b = F.Haystack.from_host(hay, buf_lo=top - n, global_len=top, own_lo=top - n + 256, own_hi=top)
    calls = [lambda h: h.search_levenshtein(pat, 2), lambda h: h.search_levenshtein(pat, 2, F.F_FORCE_DENSE),
             lambda h: h.search_levenshtein(pat, 2, F.F_TINY_LIST), lambda h: h.search_hamming(pat, 3),
             lambda h: h.search_exact(pat), lambda h: h.search_generic(pat, 2, 1, 1, 2),
             lambda h: h.search_levenshtein(pat[:8], 3), lambda h: h.search_levenshtein(pat[:4], 4)]  # LP, LP k >= m
    for ci, call in enumerate(calls):
        ra, rb = call(a), call(b)
        for which in (F.RAW, F.FINAL):
            ta, tb = sorted(ra.triples(which)), sorted(rb.triples(which))
            assert ta and [(s + top - n, e + top - n, d) for s, e, d in ta] == tb, (ci, which)
        ra.close()
        rb.close()
    a.close()
    b.close()
    for glen, blo in (((1 << 46), (1 << 46) - 4096), ((1 << 46), 0), ((1 << 64) - 1, 0)):
        with pytest.raises(ValueError, match="global_len must be below 2"):
            F.Haystack.from_host(hay, buf_lo=blo, global_len=glen, own_lo=blo, own_hi=blo + n)
