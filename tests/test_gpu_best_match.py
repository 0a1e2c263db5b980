"""best_match_in_each / fzb_best_per_record (DESIGN.md section 5.13): every sequence of a set assigned its nearest
pattern on the device.  Every case compares all six arrays, element for element, with `reduce_lists` over the dicts of
find_near_matches_batch_in_each -- the table of the semantics restated on Match lists, knowing nothing of the device's
packed words -- and, on a sample of records, with the same reduction over the oracle's lists.  `small` keeps the sizes
the CPU emulator replays (tests/test_emu_best_match.py)."""
import numpy as np
import pytest

import oracle
from corpus import ASCII, DNA, mutate
from fuzzysearch_b200 import (BestMatches, DeviceSequenceSet, Match, _native as F, best_match_in_each,
                              find_near_matches, find_near_matches_batch_in_each)
from test_gpu_records import EMU, joined, rand
from test_gpu_records_batch import GEN_MIX, lev_mix, make_set, shared_count

pytestmark = pytest.mark.gpu

NAMES = ("pattern", "start", "end", "dist", "second_pattern", "second_dist")


def reduce_lists(lists, n):
    """lists[i]: {record: its non-empty match list of pattern i} (.start / .end / .dist, or triples) -> the six
    columns of the semantics' table."""
    cols = {name: [-1] * n for name in NAMES}
    per = {}  # record -> (dist, pattern, start, end) of each pattern's best match in it
    for i, d in enumerate(lists):
        for r, ms in d.items():
            ms = [tuple(m) if isinstance(m, tuple) else (m.start, m.end, m.dist) for m in ms]
            s, e, dist = min(ms, key=lambda m: (m[2], -(m[1] - m[0]), m[0]))
            per.setdefault(r, []).append((dist, i, s, e))
    for r, rows in per.items():
        rows.sort()
        cols["dist"][r], cols["pattern"][r], cols["start"][r], cols["end"][r] = rows[0]
        if len(rows) > 1:
            cols["second_dist"][r], cols["second_pattern"][r] = rows[1][:2]
    return cols


def assert_columns(got, exp, ctx=()):
    """got: BestMatches or the binding's tuple of arrays"""
    for j, name in enumerate(NAMES):
        col = getattr(got, name) if isinstance(got, BestMatches) else got[j]
        assert col.dtype == (np.int64 if name in ("start", "end") else np.int32), name
        bad = np.flatnonzero(col != np.asarray(exp[name]))
        assert bad.size == 0, ctx + (name, bad[:5].tolist(), col[bad[:5]].tolist(), [exp[name][b] for b in bad[:5]])


def oracle_lists(pats, recs, lim, sample):
    out = []
    for q, p in enumerate(pats):
        one = {k: (v[q] if isinstance(v, list) else v) for k, v in lim.items()}
        out.append({r: ms for r in sample for ms in [oracle.find_near_matches(p, recs[r], **one)] if ms})
    return out


def check(pats, seqs, lim, resident=None, sample=None, with_oracle=True):
    """best_match_in_each == the reduction of find_near_matches_batch_in_each (and of the oracle on `sample`)."""
    target = seqs if resident is None else resident
    exp = reduce_lists(find_near_matches_batch_in_each(pats, target, **lim), len(seqs))
    got = best_match_in_each(pats, target, **lim)
    assert isinstance(got, BestMatches) and len(got) == len(seqs)
    assert_columns(got, exp, (lim,))
    if with_oracle and isinstance(seqs[0] if seqs else b"", (bytes, bytearray)):
        sample = range(len(seqs)) if sample is None else sample
        ora = reduce_lists(oracle_lists(pats, seqs, lim, sample), len(seqs))
        for name in NAMES:
            assert [getattr(got, name)[r] for r in sample] == [ora[name][r] for r in sample], (lim, name)
    return got


def kwargs4(lims4):
    s, i, d, l = zip(*lims4)
    return dict(max_substitutions=list(s), max_insertions=list(i), max_deletions=list(d), max_l_dist=list(l))


def check_handle(hs, recs, pats, lims4, flags=0):
    """The binding on a handle with the record set of `recs`: limits as the normalised 4-tuples of the C-ABI."""
    got, stats = hs.best_per_record(pats, *zip(*lims4), flags=flags)
    exp = reduce_lists(find_near_matches_batch_in_each(pats, recs, **kwargs4(lims4)), len(recs))
    assert_columns(got, exp, (flags,))
    assert stats["n_launches"] >= 1
    return got


def lev4(k):
    return (k, k, k, k)


def ham4(k):
    return (k, 0, 0, k)


def test_every_shared_pass(cuda_device, small=False):
    """q-sample, prefix and LP passes (more than 64 LP patterns), exact patterns, Hamming passes with 4-byte, 3-byte and
    2-bit keys, generic n-gram and LP passes, and a pattern of 70 bytes left to its own search -- in one call each and
    all classes mixed in one call, whose pattern order interleaves the classes."""
    rng = np.random.default_rng(131)
    pats, ks = lev_mix(rng, ASCII, 6 if small else 70)
    recs = make_set(rng, ASCII, pats, ks, small)
    buf, off = joined(recs)
    hs = F.Haystack.from_host(buf)
    hs.set_records(off)
    res, _ = hs.search_levenshtein_batch(pats, ks, F.F_PER_RECORD)
    for route in ("ngrams/sampled-filter", "ngrams/dense-filter", "lp"):
        assert shared_count(res, route) >= 1, route
    for r in res:
        r.close()
    check_handle(hs, recs, pats, [lev4(k) for k in ks])
    hs.close()
    check(pats, recs, dict(max_l_dist=ks))
    hpats = [rand(rng, ASCII, m) for m in (16, 16, 17, 24, 9, 9, 10, 12)]
    hks = [1, 1, 1, 2, 2, 2, 2, 3]
    hrecs = make_set(rng, ASCII, hpats, hks, small)
    check(hpats, hrecs, dict(max_substitutions=hks, max_insertions=0, max_deletions=0))
    dpats = [rand(rng, DNA, m) for m in (16, 18, 20, 24, 12, 24)]
    dks = [1, 1, 2, 2, 1, 3]
    drecs = make_set(rng, DNA, dpats, dks, small)
    check(dpats, drecs, dict(max_substitutions=dks, max_insertions=0, max_deletions=0))
    gpats = [rand(rng, ASCII, m) for m, _ in GEN_MIX]
    glims = [lim for _, lim in GEN_MIX]
    grecs = make_set(rng, ASCII, gpats, glims, small)
    check(gpats, grecs, kwargs4(glims))
    # all classes in one call, interleaved: no class's position in its own batch is its position in the call
    n = min(len(pats), len(hpats), len(gpats)) if small else len(gpats)
    mixed, lims4 = [], []
    for q in range(n):
        mixed += [hpats[q % len(hpats)], pats[q], gpats[q]]
        lims4 += [ham4(hks[q % len(hpats)]), lev4(ks[q]), glims[q]]
    mrecs = [hrecs[i % len(hrecs)] + grecs[i % len(grecs)] + recs[i % len(recs)][:4000] for i in range(len(recs))]
    check(mixed, mrecs, kwargs4(lims4), with_oracle=small)


def test_dna_levenshtein_pass_and_chunk_seams(cuda_device, small=False):
    """Levenshtein barcodes over DNA reads: the 2-bit n-gram pass; with FZB_F_TINY_LIST its chunks of 3 000 positions put
    seams inside reads, and its 8-hit list overflows, so the pass is redone pattern by pattern."""
    rng = np.random.default_rng(132)
    pats = [rand(rng, DNA, m) for m in (12, 12, 14, 16, 18, 20, 24, 13)]
    reads = [bytearray(rand(rng, DNA, 150)) for _ in range(60 if small else 2000)]
    for i, r in enumerate(reads):
        if i % 3:
            v = mutate(rng, pats[i % len(pats)], DNA, int(rng.integers(0, 2)))
            p = int(rng.integers(0, 150 - len(v)))
            r[p:p + len(v)] = v
    reads = [bytes(r) for r in reads]
    buf, off = joined(reads)
    hs = F.Haystack.from_host(buf)
    hs.set_records(off)
    plain = check_handle(hs, reads, pats, [lev4(1)] * len(pats))
    tiny = check_handle(hs, reads, pats, [lev4(1)] * len(pats), F.F_TINY_LIST)
    for a, b in zip(plain, tiny):
        assert np.array_equal(a, b)
    hs.close()
    check(pats, reads, dict(max_l_dist=1), sample=range(0, len(reads), 7))


def test_overflowing_passes_leave_nothing_behind(cuda_device, small=False):
    """FZB_F_TINY_LIST: the q-sample work list, the prefix pass's hit list, the LP survivor list (one 3 000-start chunk
    with more than 1 024 survivors, behind chunks that did fit) and the Hamming pass's record list overflow, and their
    patterns are searched again one by one.  The classes interleave, so a pattern's position in its pass is not its
    position in the call: a contribution kept from an abandoned pass, or one reduced under another pass's numbering,
    would name the wrong pattern.  The same handle then answers an untouched call, and ordinary batches, as before."""
    rng = np.random.default_rng(133)
    lpats, ks = lev_mix(rng, ASCII, 4)
    hpats = [rand(rng, ASCII, 16) for _ in range(4)]
    recs = make_set(rng, ASCII, lpats, ks, small)
    lp = [q for q, k in enumerate(ks) if len(lpats[q]) <= 8 and k]
    recs.append(lpats[lp[0]] * 700)
    recs.append(b"".join(lpats) * 2)
    recs += [hpats[i % 4] * 3 for i in range(40)]
    pats, lims4 = [], []
    for q in range(len(lpats)):
        pats += [hpats[q % 4][:16 - q % 3], lpats[q]]
        lims4 += [ham4(1), lev4(ks[q])]
    buf, off = joined(recs)
    hs = F.Haystack.from_host(buf)
    hs.set_records(off)
    plain = check_handle(hs, recs, pats, lims4)
    tiny = check_handle(hs, recs, pats, lims4, F.F_TINY_LIST)
    again = check_handle(hs, recs, pats, lims4)
    for a, b, c in zip(plain, tiny, again):
        assert np.array_equal(a, b) and np.array_equal(a, c)
    assert_batch_still_equals_singles(hs, lpats[:6], ks[:6])
    gpats = [rand(rng, ASCII, m) for m, _ in GEN_MIX]
    glims = [lim for _, lim in GEN_MIX]
    grecs = make_set(rng, ASCII, gpats, glims, small) + [gpats[5] * 700]
    hs.upload(joined(grecs)[0])
    hs.set_records(joined(grecs)[1])
    check_handle(hs, grecs, gpats, glims, F.F_TINY_LIST)
    hs.close()


def assert_batch_still_equals_singles(hs, pats, ks):
    res, _ = hs.search_levenshtein_batch(pats, ks, F.F_PER_RECORD)
    for p, k, r in zip(pats, ks, res):
        one = hs.search_levenshtein(p, k)
        assert r.triples(F.FINAL) == one.triples(F.FINAL)
        assert sorted(r.triples(F.RAW)) == sorted(one.triples(F.RAW))
        one.close()
        r.close()


def test_ties(cuda_device):
    A, B = b"ACGTTGCAAC", b"TTGACCAGTA"
    cases = [
        # two patterns at the same distance in one read: the smaller index wins, second_dist == dist
        ([A, B], [b"xx" + A + b"yy" + B + b"zz", b"xx" + B + b"yy" + A], dict(max_l_dist=1)),
        # duplicate patterns: index 0 wins, index 1 is the runner-up at the same distance
        ([A, A, B], [b"--" + A + b"--", b"--" + A[:4] + b"x" + A[5:] + b"--" + B], dict(max_l_dist=1)),
        # the same pattern twice in a read: no runner-up, or another pattern's
        ([A, B], [A + b"----" + A, A + b"--" + A[:3] + A[4:] + b"--" + B[:5] + b"x" + B[6:]], dict(max_l_dist=1)),
        # equal distance, different lengths (the longest), and equal length, different starts (the leftmost)
        ([b"ABCDEFGH"], [b"..ABCDEFG..ABCDEFGH..", b"..ABCDXEFGH..ABCDEFG.", b".ABCDEFG...ABCDEFG."], dict(max_l_dist=1)),
        ([b"ABCDEFGH"], [b"..ABCDEFG..ABCDEFGH..", b".ABCDEFGx...xBCDEFGH."],
         dict(max_substitutions=1, max_insertions=0, max_deletions=0)),
        # overlapping raw matches whose group winner is not the first raw record
        ([b"AAAB"], [b"AAAAAAB", b"xAAABAAAB", b"AABAAAB"], dict(max_l_dist=1)),
        ([b"ABAB", b"BABA"], [b"ABABABAB", b"xBABAx", b"ABxAB"], dict(max_l_dist=2)),
        ([b"ABCD", b"BCD"], [b"xABCDx"], dict(max_l_dist=0)),
    ]
    for pats, recs, lim in cases:
        got = check(pats, recs, lim)
        for r in range(len(recs)):
            if got.second_pattern[r] >= 0:
                assert got.second_pattern[r] != got.pattern[r] and got.second_dist[r] >= got.dist[r]
    got = check([A, B], [b"xx" + A + b"yy" + B + b"zz"], dict(max_l_dist=1))
    assert (got.pattern[0], got.dist[0], got.second_pattern[0], got.second_dist[0]) == (0, 0, 1, 0)
    got = check([A, B], [A + b"----" + A], dict(max_l_dist=1))
    assert (got.pattern[0], got.start[0], got.second_pattern[0], got.second_dist[0]) == (0, 0, -1, -1)


def test_record_edges(cuda_device, small=False):
    """Empty records, records shorter than the pattern, one-byte records, a match ending on a record's last byte,
    patterns whose max_l_dist reaches their length (an empty match (n, n, m) at every record's end position, which
    belongs to the record it closes), separators inside patterns, reads without a match."""
    rng = np.random.default_rng(134)
    P = b"GATTACAGATTACA"
    recs = [b"", b"G", P[:5], b"", b"xx" + P, P, b"q" * 70, b"", P[:-1] + b"x", b"zz" + P[1:], b"A", b""]
    recs += [rand(rng, ASCII, int(n)) for n in rng.integers(0, 200, size=8 if small else 200)]
    for lim in (dict(max_l_dist=[2, 1, 0]), dict(max_substitutions=[1, 2, 0], max_insertions=0, max_deletions=0),
                dict(max_substitutions=[1, 1, 0], max_insertions=[1, 0, 0], max_deletions=[0, 1, 0], max_l_dist=[2, 1, 0])):
        check([P, P[2:10], P[:6]], recs, lim)
    # max_l_dist >= len(pattern): every non-empty record matches, a one-byte record also at its end position
    for pats, lim in (([b"AB", b"GAT"], dict(max_l_dist=[2, 3])), ([b"ABC", b"G", P], dict(max_l_dist=[3, 1, 1])),
                      ([b"AB", b"GA"], dict(max_substitutions=[2, 1], max_insertions=[2, 2], max_deletions=[2, 2],
                                            max_l_dist=[3, 2]))):
        got = check(pats, recs, lim)
        assert all(p >= 0 for p, r in zip(got.pattern.tolist(), recs) if r)  # (empty sequences: as the class has it)
        i, m = got[1]
        assert m in find_near_matches(pats[i], recs[1], **{k: v[i] for k, v in lim.items()})
    # the separator's value inside patterns, planted across separators: whole copies inside records count, no other
    pz = [rand(rng, ASCII, 6) + b"\0" + rand(rng, ASCII, 9), rand(rng, ASCII, 3) + b"\0" + rand(rng, ASCII, 3)]
    zrecs = [bytearray(rand(rng, ASCII, n)) for n in (70, 63, 64, 65, 100, 40)]
    for i in range(len(zrecs) - 1):
        p = pz[i % 2]
        h = p.index(b"\0")
        zrecs[i][len(zrecs[i]) - h:] = p[:h]
        zrecs[i + 1][:len(p) - h - 1] = p[h + 1:]
    zrecs[2][20:20 + len(pz[0])] = pz[0]
    zrecs[4][30:30 + len(pz[1])] = pz[1]
    check(pz, [bytes(r) for r in zrecs], dict(max_l_dist=[2, 1]))
    check(pz, [bytes(r) for r in zrecs], dict(max_l_dist=0))


def test_public_api(cuda_device, small=False):
    rng = np.random.default_rng(135)
    pats = [rand(rng, ASCII, m) for m in (8, 12, 6, 20)]
    recs = make_set(rng, ASCII, pats, [2] * 4, True, extra=6)[:10 if small else 24] + [b"", b"x"]
    limits = [dict(max_l_dist=0), dict(max_l_dist=1), dict(max_l_dist=[1, 2, 0, 3]),
              dict(max_substitutions=1, max_insertions=0, max_deletions=0),
              dict(max_substitutions=[1, 1, 2, 0], max_insertions=[1, 0, 1, 0], max_deletions=[0, 0, 1, 0],
                   max_l_dist=[2, 1, 2, 0])]
    for seqs in (recs, tuple(recs), [bytearray(r) for r in recs]):
        for lim in limits:
            check(pats, seqs, lim, with_oracle=False)
    # a resident set across calls with different batches: earlier arrays stay as they were, nothing is carried over
    resident = DeviceSequenceSet(recs)
    first = check(pats, recs, limits[1], resident=resident)
    kept = [getattr(first, name).copy() for name in NAMES]
    check(pats[::-1], recs, limits[3], resident=resident)
    check(pats[:1], recs, limits[0], resident=resident)
    check([b"no such text"], recs, dict(max_l_dist=1), resident=resident)
    assert all(np.array_equal(getattr(first, name), k) for name, k in zip(NAMES, kept))
    assert_columns(best_match_in_each(pats, resident, **limits[1]), dict(zip(NAMES, kept)))
    assert find_near_matches_batch_in_each(pats, resident, max_l_dist=1) == [
        {r: ms for r, s in enumerate(recs) for ms in [find_near_matches(p, s, max_l_dist=1)] if ms} for p in pats]
    # best[r]: (pattern index, Match) with `matched` sliced from the caller's sequence, or None
    for r in range(len(recs)):
        if first.pattern[r] < 0:
            assert first[r] is None
        else:
            i, m = first[r]
            assert isinstance(m, Match) and m in find_near_matches(pats[i], recs[r], max_l_dist=1)
            assert m.matched == recs[r][m.start:m.end]
    resident.close()
    texts = [r.decode("latin-1") for r in recs]
    tpats = [p.decode("latin-1") for p in pats]
    got = check(tpats, texts, limits[2])
    hit = int(np.flatnonzero(got.pattern >= 0)[0])
    assert got[hit][1].matched == texts[hit][got.start[hit]:got.end[hit]]
    # a general-Unicode set, reduced again for each new batch alphabet
    wide = ["αβγδ" + t + "ωψ" for t in texts] + ["", "γδ€"]
    resident = DeviceSequenceSet(wide)
    for batch_pats in (["γδ" + tpats[0][:3], tpats[1]], ["€αβ", "ψ\U0001F600", tpats[2]], tpats):
        for lim in (dict(max_l_dist=1), dict(max_substitutions=1, max_insertions=0, max_deletions=0)):
            got = check(batch_pats, wide, lim, resident=resident)
            for r in np.flatnonzero(got.pattern >= 0)[:3].tolist():
                assert got[r][1].matched == wide[r][got.start[r]:got.end[r]]
    resident.close()
    # more than 255 distinct symbols over the batch: reduced on the host from the per-pattern searches
    many = ["".join(chr(0x400 + 40 * q + j) for j in range(40)) for q in range(7)]
    wide2 = [many[q % 7][5:25] + "xyz" + many[(q + 3) % 7][:12] for q in range(10)] + [""]
    check(many, wide2, dict(max_l_dist=2))
    # empty inputs and the errors of find_near_matches_batch_in_each, raised before anything is uploaded
    none = best_match_in_each([], recs, max_l_dist=1)
    assert len(none) == len(recs) and all((getattr(none, name) == -1).all() for name in NAMES) and none[0] is None
    empty = best_match_in_each(pats, [], max_l_dist=1)
    assert len(empty) == 0 and all(getattr(empty, name).shape == (0,) for name in NAMES)
    assert_columns(best_match_in_each(pats[:1], [b"", b""], max_l_dist=1), reduce_lists([{}], 2))
    with pytest.raises(ValueError, match="No limitations given!"):
        best_match_in_each(pats, recs)
    with pytest.raises(ValueError, match="Given subsequence is empty!"):
        best_match_in_each([pats[0], b""], [], max_l_dist=1)
    with pytest.raises(ValueError, match="subsequence must not be empty"):
        best_match_in_each([b""], recs, max_l_dist=0)
    with pytest.raises(ValueError, match="one max_l_dist per subsequence"):
        best_match_in_each(pats, recs, max_l_dist=[1, 2])
    with pytest.raises(TypeError):
        best_match_in_each(pats, b"not a list", max_l_dist=1)
    with pytest.raises(TypeError):
        best_match_in_each(tpats, recs, max_l_dist=1)


def test_refusals_leave_the_handle_as_it_was(cuda_device):
    rng = np.random.default_rng(136)
    pats = [rand(rng, ASCII, 24), rand(rng, ASCII, 24), rand(rng, ASCII, 7)]
    ks = [2, 2, 2]
    recs = make_set(rng, ASCII, pats, ks, True)
    buf, off = joined(recs)
    hs = F.Haystack.from_host(buf)
    lims4 = [lev4(k) for k in ks]
    hs.record_count = len(recs)  # (room for the output: the library refuses before it writes)
    with pytest.raises(ValueError, match="record set"):
        hs.best_per_record(pats, *zip(*lims4))
    res, _ = hs.search_levenshtein_batch(pats, ks)  # still a plain sequence
    for p, k, r in zip(pats, ks, res):
        assert r.triples(F.FINAL) == hs.search_levenshtein(p, k).triples(F.FINAL)
        r.close()
    hs.set_records(off)
    good = check_handle(hs, recs, pats, lims4)
    refused = [
        (F.UnsupportedError, lambda: hs.best_per_record([b"ab"] * 65536, *zip(*[lev4(0)] * 65536))),
        (F.UnsupportedError, lambda: hs.best_per_record(pats, *zip(*lims4), flags=F.F_FORCE_DENSE)),
        (F.UnsupportedError, lambda: hs.best_per_record(pats, *zip(*lims4), flags=F.F_NO_FINAL | F.F_TINY_LIST)),
        (F.UnsupportedError, lambda: hs.best_per_record(pats + [b"x" * 256], *zip(*(lims4 + [lev4(1)])))),
        (F.UnsupportedError, lambda: hs.best_per_record(pats + [b"x" * 200], *zip(*(lims4 + [(70, 0, 70, 70)])))),
        (ValueError, lambda: hs.best_per_record(pats + [b""], *zip(*(lims4 + [lev4(1)])))),
    ]
    for exc, call in refused:
        with pytest.raises(exc):
            call()
        assert_batch_still_equals_singles(hs, pats, ks)
        for a, b in zip(check_handle(hs, recs, pats, lims4), good):
            assert np.array_equal(a, b)
    hs.close()


def test_a_million_reads_and_96_barcodes(cuda_device):
    if EMU:
        pytest.skip("needs a real GPU: a million reads")
    rng = np.random.default_rng(137)
    n, length = 1 << 20, 150
    alpha = np.frombuffer(DNA, dtype=np.uint8)
    reads = alpha[rng.integers(0, 4, size=(n, length))]
    codes = [rand(rng, DNA, int(m)) for m in rng.integers(8, 25, size=96)]
    for i in range(0, n, 3):
        c = codes[int(rng.integers(0, len(codes)))]
        v = np.frombuffer(mutate(rng, c, DNA, 1), dtype=np.uint8)[:length]
        p = int(rng.integers(0, length - len(v) + 1))
        reads[i, p:p + len(v)] = v
    reads = [r.tobytes() for r in reads]
    resident = DeviceSequenceSet(reads)
    subs = [1 + (q % 2) for q in range(len(codes))]
    sample = rng.choice(n, size=300, replace=False).tolist()
    check(codes, reads, dict(max_substitutions=subs, max_insertions=0, max_deletions=0), resident=resident,
          sample=sample)
    check(codes[:16], reads, dict(max_l_dist=1), resident=resident, sample=sample)
    resident.close()


def test_two_million_lines_and_1024_mixed_terms(cuda_device):
    if EMU:
        pytest.skip("needs a real GPU: two million lines")
    rng = np.random.default_rng(138)
    n = 2_000_000
    alpha = np.frombuffer(ASCII, dtype=np.uint8)
    lengths = rng.integers(20, 120, size=n)
    flat = alpha[rng.integers(0, len(alpha), size=int(lengths.sum()))]
    ends = np.cumsum(lengths)
    terms, kw = [], dict(max_substitutions=[], max_insertions=[], max_deletions=[], max_l_dist=[])
    for q in range(1024):
        m = int(rng.integers(6, 33))
        terms.append(rand(rng, ASCII, m))
        cls = q % 4
        k = 0 if cls == 0 else 1 if m < 16 else 2
        s, i, d = [(0, 0, 0), (k, 0, 0), (k, k, k), (k, 1, 0)][cls]
        for name, v in zip(("max_substitutions", "max_insertions", "max_deletions", "max_l_dist"), (s, i, d, k)):
            kw[name].append(v)
    for r in rng.choice(n, size=n // 4, replace=False).tolist():
        v = mutate(rng, terms[int(rng.integers(0, len(terms)))], ASCII, int(rng.integers(0, 2)))
        if lengths[r] >= len(v):
            p = int(ends[r] - lengths[r] + rng.integers(0, lengths[r] - len(v) + 1))
            flat[p:p + len(v)] = np.frombuffer(v, dtype=np.uint8)
    blob = flat.tobytes()
    lines = [blob[e - l:e] for e, l in zip(ends.tolist(), lengths.tolist())]
    resident = DeviceSequenceSet(lines)
    check(terms, lines, kw, resident=resident, with_oracle=False)
    resident.close()
