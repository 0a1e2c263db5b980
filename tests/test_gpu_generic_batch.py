"""fzb_search_generic_batch: many generic-limit patterns over one resident haystack in the shared scans of the
Levenshtein batch with generic verification (DESIGN.md section 5.9), and find_near_matches_batch with all four search
classes.  Every case checks that each pattern's lists equal search_generic of the same pattern on the same handle (RAW
in its order, which sorts by anchor first; FINAL with its hulls; counts), the oracle where the size allows, and that exactly the expected
patterns took a shared pass."""
import json
import os
import sys
from collections import defaultdict

import numpy as np
import pytest

import oracle
from conftest import needs_real_gpu
from corpus import ASCII, DNA, make_corpus, mutate
from fuzzysearch_b200 import DeviceSequence, _native as F, find_near_matches, find_near_matches_batch
from parity import tup

pytestmark = pytest.mark.gpu

NG, LP = "generic-ngrams/batch-scan", "generic-lp/batch-scan"
ONE_NG, ONE_LP, EXACT = "generic-ngrams", "generic-lp", "exact"


def rand_bytes(rng, alphabet, m):
    alpha = np.frombuffer(alphabet, dtype=np.uint8)
    return bytes(alpha[rng.integers(0, len(alpha), size=m)])


def plant(hay, pos, v):
    v = v[:len(hay) - pos]
    hay[pos:pos + len(v)] = np.frombuffer(v, dtype=np.uint8)


def plant_all(rng, hay, pats, lims, alphabet, per=3):
    """`per` copies of each pattern: one exact, the others with up to max_l random edits"""
    for p, lim in zip(pats, lims):
        for c in range(per):
            v = p if c == 0 else mutate(rng, p, alphabet, int(rng.integers(0, lim[3] + 1)))
            plant(hay, int(rng.integers(0, max(1, len(hay) - len(v)))), v)


def batch(hs, pats, lims, flags=0):
    return hs.search_generic_batch(pats, *zip(*lims), flags=flags)


def raw_rows(r):
    return list(zip(*[a.tolist() for a in r.arrays(F.RAW, anchors=True)]))


def check(hs, pats, lims, results, routes, hay=None):
    """Each result equals the single search on `hs`; with `hay` (the whole sequence) also the oracle; routes[i] is
    the route pattern i must report."""
    assert len(results) == len(pats)
    for i, (p, lim, r) in enumerate(zip(pats, lims, results)):
        assert r.stats()["route"] == routes[i], (i, len(p), lim)
        one = hs.search_generic(p, *lim)
        assert r.count(F.RAW) == one.count(F.RAW) and r.count(F.FINAL) == one.count(F.FINAL), (i, len(p), lim)
        assert raw_rows(r) == raw_rows(one), (i, len(p), lim)
        assert r.group_rows().tolist() == one.group_rows().tolist(), (i, len(p), lim)
        one.close()
        if hay is not None:
            assert sorted(r.triples(F.RAW)) == sorted(tup(oracle.generic_raw(p, bytes(hay), *lim))), (i, len(p), lim)


def passes(results, route):
    """number of shared scans of `route` (a shared pass reports its scan on its first pattern only)"""
    return sum(1 for r in results if r.stats()["route"] == route and r.stats()["bytes_scanned"] > 0)


def close_all(results):
    for r in results:
        r.close()


# (m, (subs, ins, dels, max_l)) with the route each takes on text / on DNA
MIX = [
    (40, (2, 1, 1, 3), NG, ONE_NG),     # q-sample lemma holds
    (48, (1, 1, 0, 2), NG, ONE_NG),
    (16, (1, 1, 0, 2), NG, ONE_NG),     # n-gram route, lemma fails: the prefix pass
    (20, (1, 0, 1, 3), NG, ONE_NG),
    (10, (2, 0, 1, 2), NG, ONE_NG),
    (8, (1, 1, 1, 3), LP, LP),          # LP route
    (6, (1, 1, 0, 2), LP, LP),
    (12, (2, 1, 1, 4), LP, LP),
    (70, (1, 1, 0, 2), ONE_NG, ONE_NG),  # m > 64
    (12, (0, 1, 1, 0), EXACT, EXACT),   # max_l_dist == 0
    (30, (12, 1, 0, 12), ONE_LP, ONE_LP),  # LP route, m + max_l > 31
    (2, (1, 1, 1, 2), ONE_LP, ONE_LP),  # LP route, lowered max_l (2) >= m
]


def mix(rng, alphabet, text):
    pats = [rand_bytes(rng, alphabet, m) for m, _, _, _ in MIX]
    return pats, [lim for _, lim, _, _ in MIX], [t if text else d for _, _, t, d in MIX]


def haystack(rng, alphabet, n, pats, lims):
    hay = np.frombuffer(rand_bytes(rng, alphabet, n), dtype=np.uint8).copy()
    plant_all(rng, hay, pats, lims, alphabet)
    return hay


def test_ascii_and_dna_mixes(cuda_device):
    rng = np.random.default_rng(9101)
    for alphabet, text in ((ASCII, True), (DNA, False)):
        pats, lims, routes = mix(rng, alphabet, text)
        hay = haystack(rng, alphabet, 20000, pats, lims)
        hs = F.Haystack.from_host(hay)
        for _ in range(2):  # twice on the same handle
            rs, total = batch(hs, pats, lims)
            check(hs, pats, lims, rs, routes, hay=hay)
            assert passes(rs, NG) == (2 if text else 0) and passes(rs, LP) == 1
            assert all(r.count(F.RAW) >= 1 for r in rs[:8])
            close_all(rs)
        hs.close()


def test_duplicates_prefixes_and_sequence_ends(cuda_device):
    """Duplicate patterns and patterns that are prefixes of each other in one pass, matches at 0 and at N - m."""
    rng = np.random.default_rng(9102)
    n = 20000
    hay = np.frombuffer(rand_bytes(rng, ASCII, n), dtype=np.uint8).copy()
    p = rand_bytes(rng, ASCII, 40)
    for pos in (0, 777, n - 40):
        plant(hay, pos, p)
    groups = [([p, p, p[:36], p[:38]], (2, 1, 1, 3)),           # q-sample pass
              ([p[:16], p[:16], p[:18]], (1, 0, 1, 2)),          # prefix pass
              ([p[:8], p[:8], p[:7], p[-8:]], (1, 1, 1, 3))]     # LP pass
    pats = [q for g, _ in groups for q in g]
    lims = [lim for g, lim in groups for _ in g]
    routes = [NG] * 7 + [LP] * 4
    hs = F.Haystack.from_host(hay)
    for _ in range(2):
        rs, _ = batch(hs, pats, lims)
        check(hs, pats, lims, rs, routes, hay=hay)
        for r in rs[:-1]:
            starts = set(r.arrays(F.FINAL)[0].tolist())
            assert 0 in starts or 1 in starts
        assert any(e == n for e in rs[-1].arrays(F.RAW)[1].tolist())
        close_all(rs)
    hs.close()


def test_window_match_shifted_past_the_hit(cuda_device):
    """The window of an n-gram hit at p0 ends the NFA's input at p0+m+k, so it holds matches that start up to 2k after
    p0 (trailing deletions).  Here P[4] == P[0] and the text at p0 is P[0:4] + P[0:15], p0 two positions before a
    granule's end: n-gram 0 occurs at p0 and at p0+4, and (p0+4, p0+19, 2), with two trailing deletions, comes from
    the windows of four hits -- n-grams 0, 1, 2 at p0+4, p0+9, p0+14, and n-gram 0 at p0, whose window ends at p0+19.
    Every aligned word of that match aligns it with a start past p0+k, yet the q-sample pass must mark p0's granule."""
    rng = np.random.default_rng(9107)
    letters = b"abcdefghijklmnopqrstuvwxyz"
    hay = np.frombuffer(rand_bytes(rng, letters, 4096), dtype=np.uint8).copy()
    pats, sites = [], []
    for p0 in (64 * 20 + 62, 64 * 40 + 62):  # p0 = 2 mod 4: no aligned word of the match sits near p0
        p = bytearray(rand_bytes(rng, letters, 17))
        p[4] = p[0]
        if p[5] == p[1]:  # (else the aligned word at p0+2, P[2:4] + P[0:2], would be P[2:6] and mark p0 anyway)
            p[5] = letters[(letters.index(p[1]) + 1) % 26]
        p = bytes(p)
        plant(hay, p0, p[:4] + p[:15])
        pats.append(p)
        sites.append(p0)
    lims = [(0, 0, 2, 2)] * 2
    hs = F.Haystack.from_host(hay)
    for _ in range(2):
        rs, _ = batch(hs, pats, lims)
        check(hs, pats, lims, rs, [NG, NG], hay=hay)
        assert passes(rs, NG) == 1
        for r, p0 in zip(rs, sites):
            assert r.triples(F.RAW).count((p0 + 4, p0 + 19, 2)) == 4
        close_all(rs)
    hs.close()


def test_refusals_come_first(cuda_device):
    """Under FZB_F_FORCE_NGRAMS a pattern shorter than max_l_dist + 1 has an n-gram length of 0: the batch fails with
    the single search's error."""
    hs = F.Haystack.from_host(np.frombuffer(b"abcdefgh" * 64, dtype=np.uint8).copy())
    with pytest.raises(ValueError) as single:
        hs.search_generic(b"ab", 1, 1, 1, 2, F.F_FORCE_NGRAMS)
    with pytest.raises(ValueError) as many:
        batch(hs, [b"abcdefgh", b"ab"], [(1, 1, 0, 1), (1, 1, 1, 2)], F.F_FORCE_NGRAMS)
    assert str(many.value) == str(single.value)
    hs.close()


def test_batch_at_64_bit_offsets(cuda_device):
    """The same bytes as an interior shard at global offsets 0 .. 2^44: the batch at each offset is the batch at 0,
    shifted."""
    rng = np.random.default_rng(9103)
    n = 30000
    pats, lims, routes = mix(rng, ASCII, True)
    hay = haystack(rng, ASCII, n, pats, lims)
    lo, hi = 256, n - 256
    a = F.Haystack.from_host(hay, buf_lo=0, global_len=n + (1 << 20), own_lo=lo, own_hi=hi)
    ra, _ = batch(a, pats, lims)
    check(a, pats, lims, ra, routes)
    for shift in (1 << 32, (1 << 40) + 16 * 12345, 1 << 44):
        b = F.Haystack.from_host(hay, buf_lo=shift, global_len=shift + n + (1 << 20), own_lo=shift + lo,
                                 own_hi=shift + hi)
        rb, _ = batch(b, pats, lims)
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
    """A batch on each shard (halo: the longest m + max_l): the union of the shards' lists is the whole handle's
    batch, with near-matches straddling every seam.  A pattern longer than the halo fails the batch on a shard with
    the single search's error."""
    rng = np.random.default_rng(9200 + nshards)
    n = (1 << 16) + 5
    pats, lims, routes = mix(rng, ASCII, True)
    hay = haystack(rng, ASCII, n, pats, lims)
    bounds = [((n * i // nshards) // 16) * 16 for i in range(nshards)] + [n]
    for si, b in enumerate(bounds[1:-1]):
        for j, delta in enumerate((-1, -5, -12, 1)):
            q = (si + j) % 8
            plant(hay, b + delta - len(pats[q]) // 2 + 200 * j, mutate(rng, pats[q], ASCII, 1))
    whole = F.Haystack.from_host(hay)
    rw, _ = batch(whole, pats, lims)
    check(whole, pats, lims, rw, routes)
    halo = max(len(p) + lim[3] for p, lim in zip(pats, lims))
    union = [[] for _ in pats]
    for i in range(nshards):
        lo, hi = bounds[i], bounds[i + 1]
        blo = max(0, lo - halo) // 16 * 16
        bhi = min(n, hi + halo)
        hs = F.Haystack.from_host(hay[blo:bhi], buf_lo=blo, global_len=n, own_lo=lo, own_hi=hi)
        rs, _ = batch(hs, pats, lims)
        check(hs, pats, lims, rs, routes)
        for q, r in enumerate(rs):
            union[q] += r.triples(F.RAW)
        close_all(rs)
        big = rand_bytes(rng, ASCII, halo + 20)
        with pytest.raises(ValueError) as single:
            hs.search_generic(big, 1, 1, 0, 2)
        with pytest.raises(ValueError) as many:
            batch(hs, pats + [big], lims + [(1, 1, 0, 2)])
        assert str(many.value) == str(single.value)
        hs.close()
    for q, r in enumerate(rw):
        assert sorted(union[q]) == sorted(r.triples(F.RAW)), q
    close_all(rw)
    whole.close()


def test_overflows_then_a_normal_batch(cuda_device):
    """FZB_F_TINY_LIST: the q-sample work list, the prefix pass's hit list and the LP survivor list overflow, and a
    start with more than 256 live candidates overflows a candidate list; each pass's patterns then go one by one.
    A normal batch on the same handle afterwards shares its scans again (the q-sample pass's de-duplication set
    was left empty)."""
    rng = np.random.default_rng(9104)
    hay = np.frombuffer(rand_bytes(rng, ASCII, 12000), dtype=np.uint8).copy()
    qs = [rand_bytes(rng, ASCII, 40) for _ in range(6)]
    ds = [rand_bytes(rng, ASCII, 16) for _ in range(6)]
    for p in qs + ds:  # more than 8 work items / hits
        for _ in range(3):
            plant(hay, int(rng.integers(0, len(hay) - 40)), p)
    hs = F.Haystack.from_host(hay)
    for pats, lim, route in ((qs, (2, 1, 1, 3), NG), (ds, (1, 0, 1, 2), NG)):
        lims = [lim] * len(pats)
        for _ in range(2):
            rs, _ = batch(hs, pats, lims, F.F_TINY_LIST)
            check(hs, pats, lims, rs, [ONE_NG] * len(pats), hay=hay)
            close_all(rs)
            rs, _ = batch(hs, pats, lims)
            check(hs, pats, lims, rs, [route] * len(pats), hay=hay)
            close_all(rs)
    hs.close()
    # LP survivors: on DNA every start passes the counting condition of a pattern holding all four symbols
    dna = np.frombuffer(rand_bytes(rng, DNA, 6000), dtype=np.uint8).copy()
    pats = [b"ACGTAC", b"TTGCAG", b"GATCCA"]
    lims = [(1, 1, 0, 2)] * 3
    hs = F.Haystack.from_host(dna)
    for _ in range(2):
        rs, _ = batch(hs, pats, lims, F.F_TINY_LIST)
        check(hs, pats, lims, rs, [ONE_LP] * 3, hay=dna)
        close_all(rs)
        rs, _ = batch(hs, pats, lims)
        check(hs, pats, lims, rs, [LP] * 3, hay=dna)
        close_all(rs)
    hs.close()
    # candidate lists: (4, 4, 4, 8) on m = 16 has starts with more than 256 live candidates (the single search
    # repeats with 2 048-entry lists)
    pat, hay, _ = make_corpus(1, 200, DNA, 16, 4, 9)
    pats, lims = [pat, pat[:8]], [(4, 4, 4, 8), (1, 1, 0, 2)]
    hs = F.Haystack.from_host(hay)
    for _ in range(2):
        rs, _ = batch(hs, pats, lims)
        check(hs, pats, lims, rs, [ONE_LP, ONE_LP], hay=hay)
        close_all(rs)
        rs, _ = batch(hs, pats[1:] * 2, lims[1:] * 2)
        check(hs, pats[1:] * 2, lims[1:] * 2, rs, [LP, LP], hay=hay)
        close_all(rs)
    hs.close()


@pytest.mark.parametrize("count,npasses", [(65, 2), (130, 3)])
def test_lp_passes_of_64(cuda_device, count, npasses):
    rng = np.random.default_rng(9105 + count)
    pats = [rand_bytes(rng, ASCII, int(rng.integers(5, 9))) for _ in range(count)]
    lims = [(1, 1, 0, 2)] * count
    hay = haystack(rng, ASCII, 8000, pats, lims)
    hs = F.Haystack.from_host(hay)
    rs, _ = batch(hs, pats, lims)
    check(hs, pats, lims, rs, [LP] * count)
    assert passes(rs, LP) == npasses
    close_all(rs)
    hs.close()


def test_golden_generic_records_in_one_batch_per_sequence(cuda_device):
    """The generic records of the reference's recorded calls and fuzz cases, grouped by sequence: one batch per
    sequence equals the single search of each pattern, and the recorded raw stream where the record is the route the
    pattern takes."""
    here = os.path.dirname(os.path.abspath(__file__))
    groups = defaultdict(list)
    for name in ("ref_suite_calls.json", "ref_fuzz.json"):
        with open(os.path.join(here, "golden", name)) as f:
            for rec in json.load(f)["records"]:
                if rec["fn"] not in ("generic_lp_raw", "generic_ngrams_raw", "generic_raw") or "exc" in rec:
                    continue
                a = rec["args"]
                pat = bytes.fromhex(a[0])
                if not pat or len(pat) > F.FZB_MAX_PATTERN or a[5] > 63:
                    continue
                groups[a[1]].append((pat, tuple(a[2:6]), rec))
    assert groups
    shared = 0
    for hay_hex, items in groups.items():
        hay = bytes.fromhex(hay_hex)
        if not hay:
            continue
        hs = F.Haystack.from_host(hay)
        pats, lims = [p for p, _, _ in items], [lim for _, lim, _ in items]
        rs, _ = batch(hs, pats, lims)
        for (p, lim, rec), r in zip(items, rs):
            one = hs.search_generic(p, *lim)
            assert raw_rows(r) == raw_rows(one), rec
            assert r.group_rows().tolist() == one.group_rows().tolist(), rec
            one.close()
            ngrams = len(p) // (lim[3] + 1) >= 3
            if rec["fn"] == "generic_raw" or rec["fn"] == ("generic_ngrams_raw" if ngrams else "generic_lp_raw"):
                assert sorted(r.triples(F.RAW)) == sorted(tup(rec["result"])), rec
            shared += r.stats()["route"] in (NG, LP)
        close_all(rs)
        hs.close()
    assert shared > 0


LIMITS = [  # all four search classes, three generic patterns
    dict(max_l_dist=0),
    dict(max_substitutions=2, max_insertions=0, max_deletions=0),
    dict(max_l_dist=2),
    dict(max_substitutions=1, max_insertions=1, max_deletions=0, max_l_dist=2),
    dict(max_substitutions=2, max_insertions=0, max_deletions=1, max_l_dist=3),
    dict(max_substitutions=0, max_insertions=1, max_deletions=1),
]


def sequences(rng):
    """the same text as every sequence kind the package takes -> [(sequence, patterns)]"""
    base = rand_bytes(rng, ASCII[:60], 6000)
    pats = [base[100:112], base[2000:2024], base[3000:3020], base[4000:4018], base[5000:5030], base[5500:5508]]
    pats = [mutate(rng, p, ASCII[:60], 1) for p in pats]
    table = str.maketrans(ASCII[:60].decode(), "".join(chr(0x3B1 + i) for i in range(60)))
    wide = base.decode("latin-1").translate(table)
    wpats = [p.decode("latin-1").translate(table) for p in pats]
    return [(base, pats), (base.decode("latin-1"), [p.decode("latin-1") for p in pats]), (wide, wpats),
            (list(base), [list(p) for p in pats]), (DeviceSequence(base), pats)]


def test_public_api_mixes_every_search_class(cuda_device):
    rng = np.random.default_rng(9106)
    lim = {key: [d.get(key) for d in LIMITS]
           for key in ("max_substitutions", "max_insertions", "max_deletions", "max_l_dist")}
    for seq, pats in sequences(rng):
        got = find_near_matches_batch(pats, seq, **lim)
        want = [find_near_matches(p, seq, **d) for p, d in zip(pats, LIMITS)]
        assert got == want, type(seq)
        assert sum(1 for w in want if w) >= 4
        # one value for every pattern: all generic
        kw = dict(max_substitutions=1, max_insertions=1, max_deletions=0, max_l_dist=2)
        assert find_near_matches_batch(pats, seq, **kw) == [find_near_matches(p, seq, **kw) for p in pats]


def test_ascii_workload_at_4_gib(cuda_device):
    """The probe's ASCII workload (tools/probe_generic_batch.py) on 4 GiB: every list equals its single search."""
    needs_real_gpu("4 GiB haystack")
    sys.path.insert(0, os.path.join(os.path.dirname(os.path.dirname(os.path.abspath(__file__))), "tools"))
    import probe_generic_batch as P
    hs, pats, lims = P.make_haystack("ascii", 4 << 30)
    rs, _ = P.batch(hs, pats, lims)
    routes = [r.stats()["route"] for r in rs]
    assert sum(routes.count(x) for x in P.SHARED) >= len(pats) // 2
    for p, lim, r in zip(pats, lims, rs):
        one = hs.search_generic(p, *lim)
        assert P.same(P.lists(r), P.lists(one)), (p, lim)
        assert r.count(F.RAW) >= 1
        one.close()
        r.close()
    hs.close()
