"""Record sets (fzb_haystack_set_records, DESIGN.md section 5.10) and find_near_matches_in_each: one pattern over
many sequences in one device pass.  Every case checks, record by record, that the set's FINAL list equals the search
of that record uploaded alone (same handle API), that its RAW list restricted to the record and shifted equals the
single search's RAW in order, and that both equal the oracle.  `small` keeps the sizes the CPU emulator replays
(tests/test_emu_records.py)."""
import os
import threading

import numpy as np
import pytest

import oracle
from corpus import ASCII, DNA, mutate
from fuzzysearch_b200 import (DeviceSequenceSet, _native as F, find_near_matches, find_near_matches_in_each)
from parity import assert_final_parity, load_golden, tup

pytestmark = pytest.mark.gpu

EMU = os.environ.get("FZB_TEST_BACKEND") == "emu"


def rand(rng, alphabet, n):
    alpha = np.frombuffer(alphabet, dtype=np.uint8)
    return bytes(alpha[rng.integers(0, len(alpha), size=n)])


def make_records(rng, alphabet, pat, lengths, k):
    """Records of the given lengths with planted occurrences: mutated copies inside, at the start, truncated at the end,
    and occurrences split over neighbouring records (which no match may join)."""
    m = len(pat)
    recs = [bytearray(rand(rng, alphabet, n)) for n in lengths]
    for i, r in enumerate(recs):
        n = len(r)
        if n >= m + k:
            v = mutate(rng, pat, alphabet, int(rng.integers(0, k + 1)))[:n]
            pos = int(rng.integers(0, n - len(v) + 1))
            r[pos:pos + len(v)] = v
        if n >= 2:
            head = pat[int(rng.integers(0, k + 1)):][:n]  # at the start, possibly missing its first bytes
            r[:len(head)] = head
            tail = pat[:max(1, m - int(rng.integers(0, k + 1)))][-n:]  # truncated at the end
            r[n - len(tail):] = tail
        if i + 1 < len(recs) and n >= m and len(recs[i + 1]) >= m and rng.random() < 0.5:
            cut = int(rng.integers(1, m))  # straddles the separator
            r[n - cut:] = pat[:cut]
            recs[i + 1][:m - cut] = pat[cut:]
    return [bytes(r) for r in recs]


def edge_lengths(m, k, small):
    ls = [0, 1, max(m - k - 1, 0), m - 1, m, m + k, 63, 64, 65, 127, 128, 129, 0, 2 * m, 3711, 3712, 3713]
    if not small:
        ls += [8191, 8192, 8193, 1 << 20]
    return ls


def joined(recs):
    off = np.zeros(len(recs) + 1, dtype=np.uint64)
    off[1:] = np.cumsum([len(r) + 1 for r in recs])
    return b"\0".join(recs) + b"\0", off


def search(hs, kind, pat, lim, flags):
    if kind == "exact":
        return hs.search_exact(pat, flags)
    if kind == "lev":
        return hs.search_levenshtein(pat, lim, flags)
    if kind == "ham":
        return hs.search_hamming(pat, lim, flags)
    return hs.search_generic(pat, *lim, flags=flags)


def oracle_raw(kind, pat, rec, lim, flags=0):
    if kind == "lev" and flags & F.F_FORCE_LP:
        return oracle.levenshtein_lp_raw(pat, rec, lim)
    if kind == "lev" and flags & F.F_FORCE_NGRAMS:
        return oracle.levenshtein_ngrams_raw(pat, rec, lim)
    if kind == "exact":
        return oracle.levenshtein_raw(pat, rec, 0)
    if kind == "lev":
        return oracle.levenshtein_raw(pat, rec, lim)
    if kind == "ham":
        return oracle.substitutions(pat, rec, lim)
    return oracle.generic_raw(pat, rec, *lim)


def oracle_final(kind, pat, rec, lim):
    if kind == "exact":
        return oracle.find_near_matches(pat, rec, max_l_dist=0)
    if kind == "lev":
        return oracle.find_near_matches(pat, rec, max_l_dist=lim)
    if kind == "ham":
        return oracle.find_near_matches(pat, rec, max_substitutions=lim, max_insertions=0, max_deletions=0)
    return oracle.find_near_matches(pat, rec, *lim)


def split(res, which, off, anchors=False):
    """the list `which` of a record-set search, per record, shifted to record coordinates (order kept)"""
    cols = res.arrays(which, anchors=anchors)
    s = cols[0]
    rec = np.searchsorted(off.astype(np.int64), s, side="right") - 1
    out = [[] for _ in range(len(off) - 1)]
    for i, row in enumerate(zip(*[c.tolist() for c in cols])):
        r = int(rec[i])
        b = int(off[r])
        row = list(row)
        row[0] -= b
        row[1] -= b
        if anchors and row[4] >= 0:  # (-1: a list without anchors)
            row[4] -= b
        out[r].append(tuple(row))
    return out


def rows(res, which, anchors=False):
    return [tuple(r) for r in zip(*[c.tolist() for c in res.arrays(which, anchors=anchors)])]


def check_set(recs, kind, pat, lim, route, flags=0, with_oracle=True, single=None):
    """The set's lists equal, record by record, the single searches (and the oracle)."""
    buf, off = joined(recs)
    hs = F.Haystack.from_host(buf)
    hs.set_records(off)
    res = search(hs, kind, pat, lim, flags)
    assert route is None or res.stats()["route"] == route, (res.stats(), kind, lim, flags)
    raw = split(res, F.RAW, off, anchors=True)
    fin = split(res, F.FINAL, off) if not flags & F.F_NO_FINAL else None
    res.close()
    own = single is None
    if own:
        single = F.Haystack.alloc(max(max(len(r) for r in recs), 1))
    try:
        for i, r in enumerate(recs):
            single.upload(r)
            one = search(single, kind, pat, lim, flags)
            ctx = (i, len(r), kind, lim, flags)
            assert raw[i] == rows(one, F.RAW, anchors=True), ctx
            if fin is not None:
                assert fin[i] == rows(one, F.FINAL), ctx
            one.close()
            if with_oracle:
                exp_raw = sorted(tup(oracle_raw(kind, pat, r, lim, flags)))
                assert sorted(x[:3] for x in raw[i]) == exp_raw, ctx
                # (forced routes' lists may differ from the default route's; the oracle's literal grouping is
                # quadratic in the million overlapping empty matches of a 1 MiB record under k >= m)
                if fin is not None and not flags & (F.F_FORCE_LP | F.F_FORCE_NGRAMS) and len(exp_raw) < 100_000:
                    assert [x[:3] for x in fin[i]] == tup(oracle_final(kind, pat, r, lim)), ctx
    finally:
        if own:
            single.close()
    hs.close()


# (kind, alphabet, m, limit, flags, route)
ROUTES = [
    ("exact", ASCII, 12, 0, 0, "exact"),
    ("lev", ASCII, 20, 2, F.F_FORCE_SAMPLED, "ngrams/sampled-filter"),
    ("lev", DNA, 20, 2, 0, "ngrams/dense-filter"),                                 # hit list
    ("lev", DNA, 20, 2, F.F_FORCE_DENSE | F.F_TINY_LIST, "ngrams/dense-filter"),   # list overflows -> granules, sweep
    ("lev", ASCII, 20, 2, F.F_FORCE_DENSE, "ngrams/dense-filter"),
    ("lev", ASCII, 8, 2, 0, "lp"),                                                 # streaming
    ("lev", DNA, 8, 2, F.F_TINY_LIST, "lp"),                                       # survivor list overflows -> tile
    ("lev", ASCII, 8, 2, F.F_FORCE_DENSE, "lp"),                                   # tile kernel
    ("lev", ASCII, 3, 3, 0, "lp"),                                                 # k >= m
    ("lev", ASCII, 8, 2, F.F_FORCE_NGRAMS | F.F_NO_FINAL, "ngrams/dense-filter"),
    ("lev", ASCII, 20, 1, F.F_FORCE_LP, "lp"),
    ("ham", ASCII, 16, 2, 0, "hamming"),                                           # counting filter
    ("ham", DNA, 16, 1, F.F_TINY_LIST, "hamming"),
    ("ham", ASCII, 8, 2, 0, "hamming"),                                            # brute-force scan
    ("gen", ASCII, 20, (2, 1, 1, 2), 0, "generic-ngrams"),
    ("gen", DNA, 8, (1, 1, 1, 2), 0, "generic-lp"),
    ("gen", ASCII, 20, (0, 2, 2, 2), F.F_NO_FINAL, "generic-ngrams"),
]


def route_case(case, small, seed=1):
    kind, alphabet, m, lim, flags, route = case
    rng = np.random.default_rng(seed + m)
    pat = rand(rng, alphabet, m)
    k = lim if isinstance(lim, int) else lim[3]
    lengths = edge_lengths(m, k, small) + [int(x) for x in rng.integers(0, 300, size=6 if small else 40)]
    rng.shuffle(lengths)
    recs = make_records(rng, alphabet, pat, lengths, k)
    check_set(recs, kind, pat, lim, route, flags, with_oracle=True)


@pytest.mark.parametrize("case", ROUTES, ids=[f"{c[0]}-{c[5]}-{c[4]}-{len(c[1])}" for c in ROUTES])
def test_every_route_per_record(cuda_device, case, small=False):
    route_case(case, small)


def test_granule_edges_and_separators(cuda_device, small=False):
    """Record boundaries exactly on granule edges and one off, occurrences planted across every separator."""
    rng = np.random.default_rng(5)
    pat = rand(rng, ASCII, 20)
    recs = []
    for n in (63, 64, 62, 65, 127, 128, 126, 129) * (2 if small else 6):
        r = bytearray(rand(rng, ASCII, n))
        r[n - 10:] = pat[:10]  # the first half at the end ...
        recs.append(r)
    for i in range(1, len(recs)):
        recs[i][:10] = pat[10:]  # ... the second half at the start of the next record
    recs = [bytes(r) for r in recs]
    for kind, lim, flags, route in (("lev", 2, F.F_FORCE_SAMPLED, "ngrams/sampled-filter"),
                                    ("lev", 2, F.F_FORCE_DENSE, "ngrams/dense-filter"), ("ham", 2, 0, "hamming"),
                                    ("exact", 0, 0, "exact"), ("gen", (1, 1, 1, 2), 0, "generic-ngrams")):
        check_set(recs, kind, pat, lim, route, flags)
    assert find_near_matches_in_each(pat, recs, max_l_dist=2) == [[] for _ in recs]
    check_set(recs, "lev", pat[:5], 2, "lp")


def test_pattern_holding_the_separator_byte(cuda_device, small=False):
    """A pattern that contains the separator's value (0) planted ACROSS separators: the joined buffer holds it byte
    for byte, but no record does, so the record-set search must not report it.  Copies inside records count."""
    rng = np.random.default_rng(8)
    for m, half in ((20, 10), (8, 4)):
        pat = rand(rng, ASCII, half) + b"\0" + rand(rng, ASCII, m - half - 1)
        recs = []
        for n in (40, 63, 64, 65, 100, 128, 129, 31) * (2 if small else 8):
            recs.append(bytearray(rand(rng, ASCII, n)))
        for i in range(len(recs) - 1):
            recs[i][len(recs[i]) - half:] = pat[:half]  # pat[:half] + separator + pat[half+1:] spans the seam
            recs[i + 1][:m - half - 1] = pat[half + 1:]
        inner = [i for i in range(0, len(recs), 3) if len(recs[i]) >= 2 * m + half]
        for i in inner:  # whole copies inside records, 0 byte included, between the head and the tail
            recs[i][m:2 * m] = pat
        recs = [bytes(r) for r in recs]
        buf, off = joined(recs)
        plain = F.Haystack.from_host(buf)
        seams = plain.search_exact(pat).count(F.RAW)
        assert seams >= len(recs) - 1  # the buffer does hold the straddling copies
        plain.close()
        cases = [("exact", 0), ("ham", 1), ("lev", 2)] if m == 20 else [("ham", 1), ("lev", 2)]  # (m = 8: LP route)
        for kind, lim in cases:
            check_set(recs, kind, pat, lim, None)
        per = find_near_matches_in_each(pat, recs, max_l_dist=0)
        assert [i for i, x in enumerate(per) if x] == inner


def test_refusals_leave_the_handle_usable(cuda_device):
    rng = np.random.default_rng(9)
    pat = rand(rng, ASCII, 12)
    recs = make_records(rng, ASCII, pat, [40, 0, 70, 13], 1)
    buf, off = joined(recs)
    hs = F.Haystack.from_host(buf)
    plain = rows(hs.search_levenshtein(pat, 1), F.FINAL)
    for bad in ([1, len(buf)], [0, len(buf) - 1], [0, 5, 5, len(buf)], [0, 9, 3, len(buf)], [len(buf)]):
        with pytest.raises(ValueError):
            hs.set_records(bad)
    hs.set_records(off)
    per = split(hs.search_levenshtein(pat, 1), F.FINAL, off)
    with pytest.raises(F.UnsupportedError):
        hs.search_levenshtein_batch([pat, pat], [1, 1])
    with pytest.raises(F.UnsupportedError):
        hs.search_hamming_batch([pat, pat], [1, 1])
    with pytest.raises(F.UnsupportedError):
        hs.search_generic_batch([pat, pat], [1, 1], [1, 1], [1, 1], [2, 2])
    with pytest.raises(F.UnsupportedError):
        hs.has_near_match(pat, 1, 1, 1, 1)
    with pytest.raises(F.UnsupportedError):
        hs.search_exact(pat, start=0, end=10)
    with pytest.raises(F.UnsupportedError):
        hs.search_levenshtein(pat, 1, F.F_GLOBAL)
    assert split(hs.search_levenshtein(pat, 1), F.FINAL, off) == per  # still the record set
    hs.write(0, buf[:4])  # a write keeps it
    assert split(hs.search_levenshtein(pat, 1), F.FINAL, off) == per
    hs.set_records(None)  # cleared: the plain results again
    assert rows(hs.search_levenshtein(pat, 1), F.FINAL) == plain
    hs.set_records(off)
    hs.upload(buf)  # an upload clears it
    assert rows(hs.search_levenshtein(pat, 1), F.FINAL) == plain
    assert hs.has_near_match(pat, 1, 1, 1, 1) in (True, False)
    hs.close()
    shard = F.Haystack.from_host(buf[:64], global_len=128, own_lo=0, own_hi=64)
    with pytest.raises(ValueError):
        shard.set_records([0, 128])
    shard.close()


def test_scale(cuda_device):
    """200 000 reads of 150 bytes: every record equals its single search, a seeded sample the oracle."""
    if EMU:
        pytest.skip("needs a real GPU: 200 000 single searches")
    rng = np.random.default_rng(11)
    n, length = 200_000, 150
    pat = rand(rng, DNA, 20)
    alpha = np.frombuffer(DNA, dtype=np.uint8)
    reads = alpha[rng.integers(0, 4, size=(n, length))]
    for i in rng.choice(n, size=n // 20, replace=False):
        v = np.frombuffer(mutate(rng, pat, DNA, int(rng.integers(0, 3))), dtype=np.uint8)[:length]
        p = int(rng.integers(0, length - len(v) + 1))
        reads[i, p:p + len(v)] = v
    reads = [r.tobytes() for r in reads]
    hits = find_near_matches_in_each(pat, reads, max_l_dist=2)
    for i in range(n):
        assert hits[i] == find_near_matches(pat, reads[i], max_l_dist=2), i
    for i in rng.choice(n, size=300, replace=False):
        assert [(x.start, x.end, x.dist) for x in hits[i]] == tup(oracle.find_near_matches(pat, reads[i], max_l_dist=2))
    ham = find_near_matches_in_each(pat[:12], reads[:20000], max_substitutions=1, max_insertions=0, max_deletions=0)
    for i in range(20000):
        assert ham[i] == find_near_matches(pat[:12], reads[i], max_substitutions=1, max_insertions=0, max_deletions=0)


def _golden_records(stride):
    recs = load_golden("ref_suite_calls.json") + load_golden("ref_fuzz.json")
    return [r for r in recs if r["fn"] == "find_near_matches"][::stride]


def test_golden_records_over_a_set(cuda_device, stride=1):
    """Each stored find_near_matches call, searched over a set of all the golden sequences: the entry of its own
    sequence is the reference's stored result (or its exception)."""
    recs = _golden_records(stride)
    seqs = sorted(set(bytes.fromhex(r["args"][1]) for r in recs))
    where = {s: i for i, s in enumerate(seqs)}
    resident = DeviceSequenceSet(seqs)
    for rec in recs:
        a = rec["args"]
        pat, hay = bytes.fromhex(a[0]), bytes.fromhex(a[1])
        ctx = "%r" % (a,)
        if "exc" in rec:
            with pytest.raises((ValueError, TypeError)):
                find_near_matches_in_each(pat, resident, *a[2:6])
            continue
        got = find_near_matches_in_each(pat, resident, *a[2:6])
        assert len(got) == len(seqs)
        ours = [(m.start, m.end, m.dist) for m in got[where[hay]]]
        subs, ins, dels, l = oracle.normalize_params(*a[2:6])
        if l == 0 or (ins == 0 and dels == 0):
            assert ours == tup(rec["result"]), ctx
        else:
            _, raw = oracle.find_near_matches(pat, hay, *a[2:6], return_raw=True)
            assert_final_parity(ours, rec["result"], raw, ctx)
        assert got[where[hay]] == find_near_matches(pat, hay, *a[2:6]), ctx
    resident.close()


def _loop(pat, seqs, **lim):
    return [find_near_matches(pat, s, **lim) for s in seqs]


LIMITS = [dict(max_l_dist=0), dict(max_l_dist=1), dict(max_l_dist=3),
          dict(max_substitutions=1, max_insertions=0, max_deletions=0),
          dict(max_substitutions=1, max_insertions=1, max_deletions=0, max_l_dist=2)]


def test_public_api_kinds(cuda_device):
    rng = np.random.default_rng(3)
    pat = rand(rng, ASCII, 8)
    recs = make_records(rng, ASCII, pat, [0, 1, 5, 7, 8, 30, 64, 200], 2)
    variants = [recs, [bytearray(r) for r in recs], [memoryview(r) for r in recs],
                [np.frombuffer(r, dtype=np.uint8) for r in recs]]
    for seqs in variants:
        for lim in LIMITS:
            assert find_near_matches_in_each(pat, seqs, **lim) == _loop(pat, seqs, **lim), lim
    texts = [r.decode("latin-1") for r in recs]
    tpat = pat.decode("latin-1")
    for lim in LIMITS:
        assert find_near_matches_in_each(tpat, texts, **lim) == _loop(tpat, texts, **lim), lim
    wide = ["αβγδ" + t + "ωψ" for t in texts] + ["", "γδ€"]
    resident = DeviceSequenceSet(wide)
    assert len(resident) == len(wide)
    for p in ("γδ" + tpat[:3], tpat, "€αβ", "ψ\U0001F600"):  # new alphabets: the set is reduced again
        for lim in LIMITS:
            assert find_near_matches_in_each(p, resident, **lim) == _loop(p, wide, **lim), (p, lim)
    resident.close()
    latin = DeviceSequenceSet(texts)  # a pattern outside latin-1 over a latin-1 set
    assert find_near_matches_in_each("€" + tpat, latin, max_l_dist=1) == _loop("€" + tpat, texts, max_l_dist=1)
    assert find_near_matches_in_each(tpat, latin, max_l_dist=1) == _loop(tpat, texts, max_l_dist=1)
    latin.close()
    try:
        from Bio.Seq import Seq
    except ImportError:
        Seq = None
    if Seq is not None:
        bio = [Seq(t) for t in texts]
        assert find_near_matches_in_each(tpat, bio, max_l_dist=1) == _loop(tpat, bio, max_l_dist=1)
    # empty sets, empty sequences under k >= m, and the errors of find_near_matches
    assert find_near_matches_in_each(pat, [], max_l_dist=1) == []
    assert find_near_matches_in_each(b"ab", [b"", b"x"], max_l_dist=2) == _loop(b"ab", [b"", b"x"], max_l_dist=2)
    with pytest.raises(ValueError, match="No limitations given!"):
        find_near_matches_in_each(pat, recs)
    with pytest.raises(ValueError, match="Given subsequence is empty!"):
        find_near_matches_in_each(b"", recs, max_l_dist=1)
    with pytest.raises(ValueError, match="subsequence must not be empty"):
        find_near_matches_in_each(b"", recs, max_l_dist=0)
    with pytest.raises(TypeError):
        find_near_matches_in_each(pat, [b"abc", "abc"], max_l_dist=1)
    with pytest.raises(TypeError):
        find_near_matches_in_each(pat, [[1, 2, 3]], max_l_dist=1)
    with pytest.raises(TypeError):
        find_near_matches_in_each(tpat, recs, max_l_dist=1)


def test_threads_share_one_set(cuda_device, n_threads=4):
    rng = np.random.default_rng(4)
    pats = [rand(rng, DNA, 12) for _ in range(n_threads)]
    recs = make_records(rng, DNA, pats[0], [int(x) for x in rng.integers(0, 200, size=60)], 1)
    resident = DeviceSequenceSet(recs)
    want = [_loop(p, recs, max_l_dist=1) for p in pats]
    errors = []

    def work(i):
        try:
            for _ in range(3):
                assert find_near_matches_in_each(pats[i], resident, max_l_dist=1) == want[i]
        except Exception as e:  # noqa: BLE001
            errors.append(e)

    ts = [threading.Thread(target=work, args=(i,)) for i in range(n_threads)]
    for t in ts:
        t.start()
    for t in ts:
        t.join()
    assert not errors, errors
    resident.close()
