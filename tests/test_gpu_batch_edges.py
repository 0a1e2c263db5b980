"""fzb_search_levenshtein_batch at its edges: shard handles at 64-bit offsets, the union of sharded batches, the
capacity limits of the three shared passes (q-sample, dense, LP), their overflow fallbacks (FZB_F_TINY_LIST) and the
chunk seams of the LP scan.  Every pattern's lists must equal the single-pattern search on the same handle, and the
oracle where the size allows.  Each test checks which patterns went through a shared pass: a shared pass reports its
scan on its first pattern only, a pattern searched on its own reports its own scan."""
import numpy as np
import pytest

import oracle
from conftest import needs_real_gpu
from corpus import ASCII, mutate
from fuzzysearch_b200 import _native as F
from parity import tup

pytestmark = pytest.mark.gpu

SAMPLED, DENSE, LP = "ngrams/sampled-filter", "ngrams/dense-filter", "lp"
TINY_LP_CHUNK = 3000  # starts per LP scan under FZB_F_TINY_LIST (api.cu: kTinyLpChunk)
LP_CHUNK = 256 << 20  # starts per LP scan otherwise


def rand_bytes(rng, alpha, m):
    return bytes(alpha[rng.integers(0, len(alpha), size=m)])


def lp_length(rng, k):
    """A length that puts budget k on the LP route (m // (k + 1) < 3, m + k <= 31).  The tests draw budgets up to 6:
    from k = 7 on, the start of a near-match often has more live candidates than the 256 a shared LP pass holds per
    lane, and the pass then leaves all its patterns to their own searches -- correct, but not the pass these tests
    are after."""
    return int(rng.integers(k + 1, min(3 * (k + 1) - 1, 31 - k) + 1))


def mixed_patterns(rng, alpha, n_sampled=4, n_dense=3, n_lp=4):
    """Patterns for each shared pass, LP ones with k <= 4 and with k in 5..6, and two the batch searches one by one
    (m > 64; k = 0).  -> (patterns, ks, expected route of each)"""
    pats, ks, routes = [], [], []

    def add(p, k, route):
        pats.append(p)
        ks.append(k)
        routes.append(route)

    for _ in range(n_sampled):  # q-sample lemma: (m - k - 3) // 4 >= k + 1
        add(rand_bytes(rng, alpha, int(rng.integers(24, 65))), int(rng.integers(1, 3)), SAMPLED)
    for _ in range(n_dense):    # L = 3, the lemma does not hold
        add(rand_bytes(rng, alpha, int(rng.integers(12, 16))), 3, DENSE)
    for i in range(n_lp):       # m // (k + 1) < 3, m + k <= 31
        k = int(rng.integers(1, 5)) if i % 2 == 0 else int(rng.integers(5, 7))
        add(rand_bytes(rng, alpha, lp_length(rng, k)), k, LP)
    add(rand_bytes(rng, alpha, 80), 3, SAMPLED)   # m > 64: one by one
    add(rand_bytes(rng, alpha, 16), 0, "exact")   # k = 0: one by one
    return pats, ks, routes


def plant(rng, hay, pat, k, pos, alphabet=ASCII):
    v = mutate(rng, pat, alphabet, int(rng.integers(0, k + 1)))[:len(hay) - pos]
    hay[pos:pos + len(v)] = np.frombuffer(v, dtype=np.uint8)


def scans(results):
    """route -> [patterns, scans]"""
    out = {}
    for r in results:
        st = r.stats()
        e = out.setdefault(st["route"], [0, 0])
        e[0] += 1
        e[1] += st["bytes_scanned"] > 0
    return out


def raw_rows(res, route):
    """The raw stream as rows (start, end, dist, n-gram, index): in generation order on the n-gram routes, sorted
    on the LP route (its order is the reference's dict order)."""
    s, e, d, ng, ix = res.arrays(F.RAW, anchors=True)
    rows = list(zip(s.tolist(), e.tolist(), d.tolist(), ng.tolist(), ix.tolist()))
    return sorted(rows) if route == LP else rows


def check_single(hs, pats, ks, results, hay=None, final=True):
    """Each batch result equals the single-pattern search on the same handle (raw with anchors, and final); with
    `hay` (a whole-sequence handle) also the oracle."""
    for pat, k, res in zip(pats, ks, results):
        one = hs.search_levenshtein(pat, k)
        route = one.stats()["route"]
        assert res.stats()["route"] == route, (pat, k)
        assert raw_rows(res, route) == raw_rows(one, route), (pat, k, route)
        if final:
            assert res.triples(F.FINAL) == one.triples(F.FINAL), (pat, k, route)
        one.close()
        if hay is not None:
            check_oracle(pat, k, res, hay)


def check_oracle(pat, k, res, hay):
    raw = oracle.levenshtein_raw(pat, hay, k)
    if res.stats()["route"] in (LP, "exact"):
        assert sorted(res.triples(F.RAW)) == sorted(tup(raw)), (pat, k)
    else:
        assert res.triples(F.RAW) == tup(raw), (pat, k)
    if k:
        assert res.triples(F.FINAL) == tup(oracle.consolidate(raw)), (pat, k)


def assert_same_lists(ra, rb, shift=0):
    for a, b in zip(ra, rb):
        route = a.stats()["route"]
        assert b.stats()["route"] == route
        moved = [(s + shift, e + shift, d, ng, ix + shift if ix >= 0 else ix)  # (LP records have no anchor)
                 for s, e, d, ng, ix in raw_rows(a, route)]
        assert moved == raw_rows(b, route), (route, hex(shift))
        assert [(s + shift, e + shift, d) for s, e, d in a.triples(F.FINAL)] == b.triples(F.FINAL), (route, hex(shift))


def close_all(results):
    for r in results:
        r.close()


def test_batch_at_64_bit_offsets(cuda_device):
    """The same bytes as an interior shard at global offsets 0 .. 2^44 (as test_positions_are_64_bit_everywhere does
    for the single-pattern routes): the batch at each offset must be the batch at offset 0, shifted, for every
    shared pass and the one-by-one path, raw and final.  The dense and LP passes pack positions into 40 bits."""
    rng = np.random.default_rng(1040)
    n = 40000
    alpha = np.frombuffer(ASCII, dtype=np.uint8)
    hay = alpha[rng.integers(0, len(alpha), size=n)].copy()
    pats, ks, routes = mixed_patterns(rng, alpha)
    for pat, k in zip(pats, ks):
        for _ in range(3):
            plant(rng, hay, pat, k, int(rng.integers(300, n - 400)))
    lo, hi = 256, n - 256  # interior anchors, halo on both sides
    a = F.Haystack.from_host(hay, buf_lo=0, global_len=n + (1 << 20), own_lo=lo, own_hi=hi)
    ra, _ = a.search_levenshtein_batch(pats, ks)
    assert [r.stats()["route"] for r in ra] == routes
    got = scans(ra)
    assert got[SAMPLED] == [5, 2] and got[DENSE] == [3, 1] and got[LP] == [4, 1] and got["exact"] == [1, 1], got
    check_single(a, pats, ks, ra)
    assert sum(r.count(F.RAW) for r in ra) >= 3 * len(pats)
    for shift in (1 << 32, (1 << 35) - 4096, (1 << 40) + 16 * 12345, 1 << 44):
        b = F.Haystack.from_host(hay, buf_lo=shift, global_len=shift + n + (1 << 20), own_lo=shift + lo,
                                 own_hi=shift + hi)
        rb, _ = b.search_levenshtein_batch(pats, ks)
        assert scans(rb) == got
        assert_same_lists(ra, rb, shift)
        close_all(rb)
        b.close()
    close_all(ra)
    a.close()


@pytest.mark.parametrize("nshards", [2, 3, 7])
def test_batch_sharded_union_equals_whole(cuda_device, nshards):
    """A batch on each shard (16-aligned seams, halo >= the largest m + k): the union of the shards' raw streams is
    the whole handle's batch.  Near-matches of patterns of every pass sit at every seam, at the deltas of
    test_sharded_union_equals_whole.  A pattern whose m + k exceeds the halo fails the batch on a shard exactly as
    it fails the single-pattern search there."""
    rng = np.random.default_rng(500 + nshards)
    n = (1 << 17) + 5
    alpha = np.frombuffer(ASCII, dtype=np.uint8)
    hay = alpha[rng.integers(0, len(alpha), size=n)].copy()
    pats, ks, routes = mixed_patterns(rng, alpha)
    for pat, k in zip(pats, ks):
        for _ in range(4):
            plant(rng, hay, pat, k, int(rng.integers(100, n - 200)))
    bounds = [((n * i // nshards) // 16) * 16 for i in range(nshards)] + [n]
    for si, b in enumerate(bounds[1:-1]):
        for j in range(7):  # seven patterns (of all passes) around the seam, one exactly across it
            q = (si + j) % len(pats)
            m = len(pats[q])
            delta = (-m, -m + 1, -4, -2, -1, 0, 1)[j]
            plant(rng, hay, pats[q], ks[q], b + delta + 96 * (j - 3))
    whole = F.Haystack.from_host(hay)
    rw, _ = whole.search_levenshtein_batch(pats, ks)
    assert [r.stats()["route"] for r in rw] == routes
    assert scans(rw)[LP] == [4, 1] and scans(rw)[SAMPLED] == [5, 2] and scans(rw)[DENSE] == [3, 1]
    check_single(whole, pats, ks, rw, hay=hay)
    halo = max(len(p) + k for p, k in zip(pats, ks))
    big, kbig = rand_bytes(rng, alpha, 110), 12  # m + k > halo + 15
    union = [[] for _ in pats]
    for i in range(nshards):
        lo, hi = bounds[i], bounds[i + 1]
        blo = max(0, lo - halo) // 16 * 16
        bhi = min(n, hi + halo)
        hs = F.Haystack.from_host(hay[blo:bhi], buf_lo=blo, global_len=n, own_lo=lo, own_hi=hi)
        rs, _ = hs.search_levenshtein_batch(pats, ks)
        assert [r.stats()["route"] for r in rs] == routes
        assert scans(rs)[LP][1] == 1 and scans(rs)[DENSE][1] == 1
        check_single(hs, pats, ks, rs, final=False)
        for q, r in enumerate(rs):
            union[q] += raw_rows(r, LP)  # (sorted)
        close_all(rs)
        with pytest.raises(ValueError) as single:
            hs.search_levenshtein(big, kbig)
        with pytest.raises(ValueError) as batch:
            hs.search_levenshtein_batch(pats + [big], ks + [kbig])
        assert str(batch.value) == str(single.value)
        hs.close()
    for q, r in enumerate(rw):
        got = sorted(union[q], key=lambda t: (t[3], t[4], t[0], t[1], t[2]))
        want = raw_rows(r, routes[q])
        if routes[q] in (LP, "exact"):
            assert sorted(got) == sorted(want), (q, routes[q])
        else:
            assert got == want, (q, routes[q])
    close_all(rw)
    whole.close()


def run_twice(hs, pats, ks, flags=0):
    """The batch, then the same batch again on the same handle: the second must equal the first (the pass left its
    de-duplication set empty).  -> the first results"""
    r1, _ = hs.search_levenshtein_batch(pats, ks, flags)
    r2, _ = hs.search_levenshtein_batch(pats, ks, flags)
    assert scans(r2) == scans(r1)
    assert_same_lists(r1, r2)
    close_all(r2)
    return r1


@pytest.mark.parametrize("count", [64, 65, 130])
def test_batch_lp_pass_limits(cuda_device, count):
    """LP-route patterns share scans of 64: 64 patterns take one pass, the 65th is searched alone (a pass of one is
    not worth it), 130 take three passes.  Budgets 5..6 (k_lp_verify_multi<8>) are mixed into the pass of 64; the
    first pass of 65 and of 130 has budgets k <= 4 only (<4>), the later ones both."""
    rng = np.random.default_rng(count)
    n = 20000
    alpha = np.frombuffer(ASCII, dtype=np.uint8)
    hay = alpha[rng.integers(0, len(alpha), size=n)].copy()
    pats, ks = [], []
    for i in range(count):
        k = int(rng.integers(1, 5)) if i < 64 or i % 2 else int(rng.integers(5, 7))
        if count == 64 and i % 3 == 0:
            k = int(rng.integers(5, 7))
        m = lp_length(rng, k)
        pats.append(rand_bytes(rng, alpha, m))
        ks.append(k)
        plant(rng, hay, pats[-1], k, int(rng.integers(50, n - 100)))
    hs = F.Haystack.from_host(hay)
    res = run_twice(hs, pats, ks)
    assert scans(res) == {LP: [count, {64: 1, 65: 2, 130: 3}[count]]}
    check_single(hs, pats, ks, res)
    for q in range(0, count, 4):
        check_oracle(pats[q], ks[q], res[q], hay)
    close_all(res)
    hs.close()


def test_batch_two_q_sample_passes(cuda_device):
    """1 000 patterns of 64 bytes have more distinct 4-grams than one q-sample pass takes (kMaxBatchGrams): two
    passes, the second one behind a pass that must have left the de-duplication set empty."""
    rng = np.random.default_rng(1000)
    n = 1 << 16
    alpha = np.frombuffer(ASCII, dtype=np.uint8)
    hay = alpha[rng.integers(0, len(alpha), size=n)].copy()
    pats = [rand_bytes(rng, alpha, 64) for _ in range(1000)]
    ks = [int(rng.integers(1, 4)) for _ in pats]
    for q in list(range(0, 1000, 10)) + list(range(983, 1000)):  # every tenth, and the whole second pass
        plant(rng, hay, pats[q], ks[q], int(rng.integers(100, n - 200)))
    hs = F.Haystack.from_host(hay)
    res = run_twice(hs, pats, ks)
    assert scans(res) == {SAMPLED: [1000, 2]}
    assert sum(r.count(F.FINAL) for r in res[983:]) >= 17
    check_single(hs, pats, ks, res)
    for q in sorted(set(rng.choice(1000, size=48, replace=False).tolist()) | set(range(983, 999))):
        check_oracle(pats[q], ks[q], res[q], hay)
    close_all(res)
    hs.close()


def test_batch_gram_with_more_than_255_postings(cuda_device):
    """The 4-gram "aaaa" has 533 postings: three slots of the gram table (255 each).  Patterns whose only 4-gram it
    is sit in the second and third slot, so every slot must be probed; the text has long runs of "a"."""
    rng = np.random.default_rng(255)
    n = 1 << 16
    alpha = np.frombuffer(ASCII, dtype=np.uint8)
    hay = alpha[rng.integers(0, len(alpha), size=n)].copy()
    pats, ks = [], []
    for i in range(4):  # 57 postings each, at offsets 0 .. 56
        pats.append(b"a" * 60 + rand_bytes(rng, alpha, 4))
        ks.append(i % 2 + 1)
    for k in (1, 2, 3, 4, 2):  # 61 postings each
        pats.append(b"a" * 64)
        ks.append(k)
    for i in range(6):  # one more shared gram "QZqz" at many offsets
        p = bytearray(rand_bytes(rng, alpha, 48))
        for o in range(i, 44, 11):
            p[o:o + 4] = b"QZqz"
        pats.append(bytes(p))
        ks.append(2)
    for q, (pat, k) in enumerate(zip(pats, ks)):
        plant(rng, hay, pat, k, 1000 + 700 * q)
    for r in range(12):
        pos = 20000 + 2000 * r
        hay[pos:pos + 70 + 10 * r] = ord("a")
    hs = F.Haystack.from_host(hay)
    res = run_twice(hs, pats, ks)
    assert scans(res) == {SAMPLED: [len(pats), 1]}
    for r in res[4:9]:
        assert r.count(F.FINAL) >= 12
    check_single(hs, pats, ks, res, hay=hay)
    close_all(res)
    hs.close()


def test_batch_overflow_fallbacks(cuda_device):
    """FZB_F_TINY_LIST: the q-sample work list (8 items), the dense pass's hit list (8 hits) and the LP survivor list
    (1 024 per chunk) all overflow, and every pattern falls back to its own search.  A normal batch of the same
    patterns right after must be correct too: the overflowing q-sample pass left entries in the de-duplication set,
    which must have been cleared."""
    rng = np.random.default_rng(808)
    n = 1 << 16
    alpha = np.frombuffer(ASCII, dtype=np.uint8)
    hay = alpha[rng.integers(0, len(alpha), size=n)].copy()
    pats, ks, routes = mixed_patterns(rng, alpha)
    for pat, k in zip(pats, ks):
        for _ in range(6):
            plant(rng, hay, pat, k, int(rng.integers(100, n - 200)))
    lp = [q for q, r in enumerate(routes) if r == LP]
    hay[30000:30000 + 2 * TINY_LP_CHUNK] = np.frombuffer((pats[lp[0]] * 2 * TINY_LP_CHUNK)[:2 * TINY_LP_CHUNK],
                                                       dtype=np.uint8)  # > 1 024 survivors in a chunk
    hs = F.Haystack.from_host(hay)
    tiny, _ = hs.search_levenshtein_batch(pats, ks, F.F_TINY_LIST)
    assert [r.stats()["route"] for r in tiny] == routes
    assert all(r.stats()["bytes_scanned"] == n for r in tiny)  # every pattern searched on its own
    check_single(hs, pats, ks, tiny, hay=hay)
    normal, _ = hs.search_levenshtein_batch(pats, ks)
    got = scans(normal)
    assert got[SAMPLED] == [5, 2] and got[DENSE] == [3, 1] and got[LP] == [4, 1], got
    assert_same_lists(tiny, normal)
    close_all(tiny)
    close_all(normal)
    hs.close()


def test_batch_lp_chunk_seams(cuda_device):
    """FZB_F_TINY_LIST scans the LP starts in chunks of 3 000 (not a multiple of the 128-byte tile rows): at every
    seam an exact occurrence starts at the last start of a chunk (straddling the seam) or at the first start of the
    next one, with more occurrences shortly before and after."""
    rng = np.random.default_rng(3000)
    n = 7 * TINY_LP_CHUNK + 123
    alpha = np.frombuffer(ASCII, dtype=np.uint8)
    hay = alpha[rng.integers(0, len(alpha), size=n)].copy()
    pats, ks = [], []
    for i in range(6):
        k = 1 + i % 4 if i < 4 else 5 + (i - 4)
        m = lp_length(rng, k)
        pats.append(rand_bytes(rng, alpha, m))
        ks.append(k)
    for c in range(1, 7):
        seam = c * TINY_LP_CHUNK
        for j, off in enumerate((-1 if c % 2 else 0, -100, 64)):
            p = pats[(c + j) % len(pats)]
            hay[seam + off:seam + off + len(p)] = np.frombuffer(p, dtype=np.uint8)
    hs = F.Haystack.from_host(hay)
    res = run_twice(hs, pats, ks, F.F_TINY_LIST)
    assert scans(res) == {LP: [len(pats), 1]}
    again, st = hs.search_levenshtein_batch(pats, ks, F.F_TINY_LIST)
    chunks = (n + TINY_LP_CHUNK - 1) // TINY_LP_CHUNK
    assert st["n_launches"] == 4 * chunks  # four launches per chunk
    assert again[0].stats()["n_launches"] == 4 * chunks  # reported by the pass, on its first result
    close_all(again)
    starts = {s for r in res for s, _, _ in r.triples(F.RAW)}
    for c in range(1, 7):
        assert c * TINY_LP_CHUNK - (1 if c % 2 else 0) in starts and c * TINY_LP_CHUNK - 100 in starts
    check_single(hs, pats, ks, res, hay=hay)
    close_all(res)
    hs.close()


def test_batch_lp_chunk_seams_at_full_size(cuda_device):
    """The LP scan's real chunks of 256 Mi starts: matches across the seams at 256 MiB and 512 MiB of a 600 MiB
    sequence, checked against the single-pattern searches over the whole sequence and the oracle around the seams."""
    needs_real_gpu("600 MiB input")
    rng = np.random.default_rng(600)
    n = 600 << 20
    alpha = np.frombuffer(ASCII, dtype=np.uint8)
    pats, ks = [], []
    for i in range(8):
        k = 1 + i % 4 if i < 6 else 5 + i % 2
        m = int(rng.integers(2 * (k + 1), min(3 * (k + 1) - 1, 31 - k) + 1))  # (m - k >= k + 2: rare on this text)
        pats.append(rand_bytes(rng, alpha, m))
        ks.append(k)
    hs = F.Haystack.alloc(n)
    hs.fill_synthetic(ASCII, 17)
    seams = (LP_CHUNK, 2 * LP_CHUNK)
    for si, seam in enumerate(seams):  # the last start of the first chunk (straddling), the first of the third
        for j, off in enumerate((-1 if si == 0 else 0, -100, 64)):
            hs.write(seam + off, pats[(si * 3 + j) % len(pats)])
    res = run_twice(hs, pats, ks)
    assert scans(res) == {LP: [len(pats), 1]}
    check_single(hs, pats, ks, res)
    starts = {s for r in res for s, _, _ in r.triples(F.RAW)}
    assert seams[0] - 1 in starts and seams[1] in starts
    for seam in seams:
        assert seam - 100 in starts and seam + 64 in starts
        lo, hi = seam - 4096, seam + 4096
        window = np.frombuffer(hs.read(lo, hi - lo), dtype=np.uint8)
        for pat, k, r in zip(pats, ks, res):
            # a start's LP matches depend on the bytes from the start on only: compare the starts well inside
            want = sorted((s + lo, e + lo, d) for s, e, d in tup(oracle.levenshtein_raw(pat, window, k))
                          if s < hi - lo - 64)
            got = sorted(t for t in r.triples(F.RAW) if lo <= t[0] < hi - 64)
            assert got == want, (pat, k, seam)
    close_all(res)
    hs.close()
