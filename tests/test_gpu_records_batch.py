"""Batches over record sets (FZB_F_PER_RECORD, DESIGN.md section 5.11) and find_near_matches_batch_in_each: many
patterns over many sequences in shared scans.  Every case checks, pattern by pattern and record by record, that the
batch's RAW list (in order; sorted on the LP routes, whose order is the reference's dict order) and FINAL list equal
the single search of that pattern on the same record set, that both equal the oracle on the record alone, and that
the intended shared pass ran (a shared pass reports its scan on its first pattern only, the others report no bytes).
`small` keeps the sizes the CPU emulator replays (tests/test_emu_records_batch.py)."""
import numpy as np
import pytest

import oracle
from corpus import ASCII, DNA, mutate
from fuzzysearch_b200 import (DeviceSequenceSet, _native as F, find_near_matches, find_near_matches_batch_in_each,
                              find_near_matches_in_each)
from parity import load_golden, tup
from test_gpu_records import EMU, edge_lengths, joined, oracle_final, oracle_raw, rand, rows, search, split

pytestmark = pytest.mark.gpu

LP_ROUTES = ("lp", "generic-lp", "generic-lp/batch-scan")
ORACLE_MAX = 1 << 16  # longer records (the 1 MiB one) are checked against the single search only


def batch(hs, kind, pats, lims, flags):
    if kind == "lev":
        return hs.search_levenshtein_batch(pats, lims, flags)
    if kind == "ham":
        return hs.search_hamming_batch(pats, lims, flags)
    return hs.search_generic_batch(pats, *zip(*lims), flags=flags)


def plant(rng, recs, pats, lims, alphabet, per=4):
    """Mutated copies of every pattern inside records, at a record's start, truncated at its end, and straddling a
    separator (which no match may join)."""
    for pat, lim in zip(pats, lims):
        k = lim if isinstance(lim, int) else lim[3]
        m = len(pat)
        for _ in range(per):
            r = recs[int(rng.integers(0, len(recs)))]
            n = len(r)
            if n >= m + k:
                v = mutate(rng, pat, alphabet, int(rng.integers(0, k + 1)))[:n]
                pos = int(rng.integers(0, n - len(v) + 1))
                r[pos:pos + len(v)] = v
        for where in ("start", "end", "seam"):
            i = int(rng.integers(0, len(recs) - 1))
            r, nxt = recs[i], recs[i + 1]
            if len(r) < m or len(nxt) < m:
                continue
            if where == "start":
                head = pat[int(rng.integers(0, k + 1)):]
                r[:len(head)] = head
            elif where == "end":
                tail = pat[:max(1, m - int(rng.integers(0, k + 1)))]
                r[len(r) - len(tail):] = tail
            else:
                cut = int(rng.integers(1, m))
                r[len(r) - cut:] = pat[:cut]
                nxt[:m - cut] = pat[cut:]


def make_set(rng, alphabet, pats, lims, small, extra=12):
    m = max(len(p) for p in pats)
    k = max(x if isinstance(x, int) else x[3] for x in lims)
    lengths = edge_lengths(m, k, small) + [int(x) for x in rng.integers(0, 300, size=extra if small else 4 * extra)]
    rng.shuffle(lengths)
    recs = [bytearray(rand(rng, alphabet, n)) for n in lengths]
    plant(rng, recs, pats, lims, alphabet)
    return [bytes(r) for r in recs]


def shared_count(results, route):
    """patterns of `route` that rode on another pattern's scan"""
    return sum(1 for r in results if r.stats()["route"] == route and r.stats()["bytes_scanned"] == 0)


def check_batch(recs, kind, pats, lims, flags=0, shared=(), with_oracle=True, hs=None):
    """The batch with FZB_F_PER_RECORD on a record set of `recs` equals, per pattern and record, the single search on
    the same set and the oracle on the record; every route of `shared` had at least one pattern riding on a shared
    scan.  -> the per-pattern (raw, final) lists per record."""
    buf, off = joined(recs)
    own = hs is None
    if own:
        hs = F.Haystack.from_host(buf)
        hs.set_records(off)
    results, _ = batch(hs, kind, pats, lims, flags | F.F_PER_RECORD)
    for route in shared:
        assert shared_count(results, route) >= 1, (route, [r.stats() for r in results])
    lists = []
    for q, (pat, lim, res) in enumerate(zip(pats, lims, results)):
        one = search(hs, kind, pat, lim, 0)
        route = one.stats()["route"]
        ctx = (q, len(pat), kind, lim, flags, route)
        raw_b, raw_1 = split(res, F.RAW, off, anchors=True), split(one, F.RAW, off, anchors=True)
        fin_b, fin_1 = split(res, F.FINAL, off), split(one, F.FINAL, off)
        if route in LP_ROUTES or kind == "ham":
            raw_b, raw_1 = [sorted(x) for x in raw_b], [sorted(x) for x in raw_1]
        assert raw_b == raw_1, ctx
        assert fin_b == fin_1, ctx
        one.close()
        res.close()
        if with_oracle:
            # (a limit of 0 is the exact search, whose list find_near_matches returns unconsolidated: RAW only)
            total = lim if isinstance(lim, int) else lim[3]
            for i, r in enumerate(recs):
                if len(r) > ORACLE_MAX:
                    continue
                exp = sorted(tup(oracle_raw(kind, pat, r, lim)))
                assert sorted(x[:3] for x in raw_b[i]) == exp, ctx + (i, len(r))
                if total:
                    assert [x[:3] for x in fin_b[i]] == tup(oracle_final(kind, pat, r, lim)), ctx + (i, len(r))
        lists.append((raw_b, fin_b))
    if own:
        hs.close()
    return lists


def lev_mix(rng, alphabet, n_lp):
    """q-sample (m 24..40, k 2), prefix (m 12..16, k 2) and LP (m 6..8, k 2) patterns, exact ones mixed in"""
    pats, ks = [], []
    for m, k, n in ((32, 2, 3), (24, 2, 2), (40, 3, 2), (14, 2, 3), (12, 2, 2), (7, 2, n_lp // 2),
                    (8, 2, n_lp - n_lp // 2), (10, 0, 2)):
        for _ in range(n):
            pats.append(rand(rng, alphabet, m))
            ks.append(k)
    return pats, ks


def test_levenshtein_passes_per_record(cuda_device, small=False):
    rng = np.random.default_rng(21)
    pats, ks = lev_mix(rng, ASCII, 6 if small else 70)  # (70: more than 64 LP patterns, two LP passes)
    recs = make_set(rng, ASCII, pats, ks, small)
    check_batch(recs, "lev", pats, ks, shared=("ngrams/sampled-filter", "ngrams/dense-filter", "lp"),
                with_oracle=True)


def test_hamming_passes_per_record(cuda_device, small=False):
    rng = np.random.default_rng(22)
    # text: 4-byte keys (pieces of 8), 3-byte keys (pieces of 3)
    pats = [rand(rng, ASCII, m) for m in (16, 16, 17, 24, 9, 9, 10, 12)]
    ks = [1, 1, 1, 2, 2, 2, 2, 3]
    recs = make_set(rng, ASCII, pats, ks, small)
    check_batch(recs, "ham", pats, ks, shared=("hamming/batch-scan",))
    # DNA: 2-bit keys
    pats = [rand(rng, DNA, m) for m in (16, 18, 20, 24, 12, 24)]
    ks = [1, 1, 2, 2, 1, 3]
    recs = make_set(rng, DNA, pats, ks, small)
    check_batch(recs, "ham", pats, ks, shared=("hamming/batch-scan",))


GEN_MIX = [(40, (2, 1, 1, 3)), (48, (1, 1, 0, 2)), (16, (1, 1, 0, 2)), (20, (1, 0, 1, 3)), (10, (2, 0, 1, 2)),
           (8, (1, 1, 1, 3)), (6, (1, 1, 0, 2)), (12, (2, 1, 1, 4)), (12, (0, 1, 1, 0)), (70, (1, 1, 0, 2))]


def test_generic_passes_per_record(cuda_device, small=False):
    rng = np.random.default_rng(23)
    pats = [rand(rng, ASCII, m) for m, _ in GEN_MIX]
    lims = [lim for _, lim in GEN_MIX]
    recs = make_set(rng, ASCII, pats, lims, small)
    check_batch(recs, "gen", pats, lims, shared=("generic-ngrams/batch-scan", "generic-lp/batch-scan"))


def test_pattern_holding_the_separator_byte(cuda_device, small=False):
    """Patterns that contain the separator's value (0), planted across every separator: the joined buffer holds
    them byte for byte, no record does.  Whole copies inside records count."""
    rng = np.random.default_rng(24)
    pats = [rand(rng, ASCII, 10) + b"\0" + rand(rng, ASCII, 21), rand(rng, ASCII, 12) + b"\0" + rand(rng, ASCII, 19),
            rand(rng, ASCII, 4) + b"\0" + rand(rng, ASCII, 3), rand(rng, ASCII, 3) + b"\0" + rand(rng, ASCII, 3)]
    recs = [bytearray(rand(rng, ASCII, n)) for n in (70, 63, 64, 65, 100, 128, 129, 90) * (2 if small else 6)]
    for i in range(len(recs) - 1):
        p = pats[i % len(pats)]
        h = p.index(b"\0")
        recs[i][len(recs[i]) - h:] = p[:h]
        recs[i + 1][:len(p) - h - 1] = p[h + 1:]
    for i in range(0, len(recs), 3):
        p = pats[i % len(pats)]
        recs[i][34:34 + len(p)] = p
    recs = [bytes(r) for r in recs]
    check_batch(recs, "lev", pats, [2, 2, 2, 2], shared=("ngrams/sampled-filter", "lp"))
    check_batch(recs, "lev", pats, [0, 0, 0, 0])
    check_batch(recs, "ham", pats[:2], [1, 1], shared=("hamming/batch-scan",))


def test_overflow_fallbacks_and_repeats(cuda_device, small=False):
    """FZB_F_TINY_LIST | FZB_F_PER_RECORD: the q-sample work list, the prefix pass's hit list, the LP survivor list and
    the Hamming pass's record list overflow and every pattern falls back to its own search; the lists still equal.
    The same batch twice on one handle after that: the overflowing q-sample pass left the de-duplication set empty."""
    rng = np.random.default_rng(25)
    pats, ks = lev_mix(rng, ASCII, 4)
    recs = make_set(rng, ASCII, pats, ks, small)
    lp = [q for q, k in enumerate(ks) if len(pats[q]) <= 8 and k]
    recs.append(pats[lp[0]] * 700)  # > 1 024 LP survivors in one 3 000-start chunk
    recs.append(b"".join(pats) * 2)  # more than 8 work items and hits
    buf, off = joined(recs)
    hs = F.Haystack.from_host(buf)
    hs.set_records(off)
    tiny = check_batch(recs, "lev", pats, ks, F.F_TINY_LIST, hs=hs, with_oracle=False)
    res, _ = hs.search_levenshtein_batch(pats, ks, F.F_TINY_LIST | F.F_PER_RECORD)
    assert all(r.stats()["bytes_scanned"] > 0 for r in res)  # every pattern on its own
    for r in res:
        r.close()
    for _ in range(2):
        assert check_batch(recs, "lev", pats, ks, hs=hs, with_oracle=False,
                           shared=("ngrams/sampled-filter", "ngrams/dense-filter", "lp")) == tiny
    hpats = [rand(rng, ASCII, 16) for _ in range(4)]
    hrecs = [hpats[i % 4] * 3 for i in range(40)]  # more than 8 records in the pass
    check_batch(hrecs, "ham", hpats, [1] * 4, F.F_TINY_LIST)
    gpats = [rand(rng, ASCII, m) for m, _ in GEN_MIX]
    glims = [lim for _, lim in GEN_MIX]
    grecs = make_set(rng, ASCII, gpats, glims, small) + [gpats[5] * 700]
    check_batch(grecs, "gen", gpats, glims, F.F_TINY_LIST, with_oracle=False)
    hs.close()


def test_refusals(cuda_device):
    rng = np.random.default_rng(26)
    pats = [rand(rng, ASCII, 24), rand(rng, ASCII, 24)]
    recs = make_set(rng, ASCII, pats, [2, 2], True)
    buf, off = joined(recs)
    hs = F.Haystack.from_host(buf)
    plain = rows(hs.search_levenshtein(pats[0], 2), F.FINAL)
    for fn in (lambda: hs.search_levenshtein_batch(pats, [2, 2], F.F_PER_RECORD),
               lambda: hs.search_hamming_batch(pats, [2, 2], F.F_PER_RECORD),
               lambda: hs.search_generic_batch(pats, [1, 1], [1, 1], [1, 1], [2, 2], flags=F.F_PER_RECORD)):
        with pytest.raises(ValueError):  # the flag needs a record set
            fn()
    assert rows(hs.search_levenshtein(pats[0], 2), F.FINAL) == plain  # left as it was
    res, _ = hs.search_levenshtein_batch(pats, [2, 2])
    assert rows(res[0], F.FINAL) == plain
    for r in res:
        r.close()
    hs.set_records(off)
    with pytest.raises(F.UnsupportedError):  # no flag: refused as before
        hs.search_levenshtein_batch(pats, [2, 2])
    with pytest.raises(F.UnsupportedError):
        hs.search_levenshtein(pats[0], 2, F.F_GLOBAL | F.F_PER_RECORD)
    # other flags with FZB_F_PER_RECORD: one by one, still per record
    for kind, lims, flags in (("lev", [2, 2], F.F_FORCE_DENSE), ("lev", [2, 2], F.F_NO_FINAL),
                              ("ham", [2, 2], F.F_FORCE_NGRAMS), ("gen", [(1, 1, 1, 2)] * 2, F.F_NO_FINAL)):
        results, _ = batch(hs, kind, pats, lims, flags | F.F_PER_RECORD)
        assert all(r.stats()["bytes_scanned"] > 0 for r in results), (kind, flags)
        for pat, lim, r in zip(pats, lims, results):
            one = search(hs, kind, pat, lim, flags)
            assert split(r, F.RAW, off) == split(one, F.RAW, off), (kind, flags)
            for i, rec in enumerate(recs):
                got = sorted(x[:3] for x in split(r, F.RAW, off)[i])
                assert got == sorted(tup(oracle_raw(kind, pat, rec, lim, flags))), (kind, flags, i)
            one.close()
            r.close()
    hs.close()
    shard = F.Haystack.from_host(buf[:64], global_len=128, own_lo=0, own_hi=64)
    with pytest.raises(ValueError):
        shard.set_records([0, 128])
    with pytest.raises(ValueError):
        shard.search_levenshtein_batch(pats, [2, 2], F.F_PER_RECORD)
    shard.close()


LIMITS = [dict(max_l_dist=0), dict(max_l_dist=1), dict(max_l_dist=[1, 2, 0, 3]),
          dict(max_substitutions=1, max_insertions=0, max_deletions=0),
          dict(max_substitutions=[1, 1, 2, 0], max_insertions=[1, 0, 1, 0], max_deletions=[0, 0, 1, 0],
               max_l_dist=[2, 1, 2, 0])]


def _each(pats, seqs, lim):
    """-> per pattern, {sequence index: find_near_matches(...)} over the sequences that hold matches"""
    out = []
    for q, p in enumerate(pats):
        one = {k: (v[q] if isinstance(v, list) else v) for k, v in lim.items()}
        out.append({r: ms for r, s in enumerate(seqs) for ms in [find_near_matches(p, s, **one)] if ms})
    return out


def test_public_api(cuda_device, small=False):
    rng = np.random.default_rng(27)
    pats = [rand(rng, ASCII, m) for m in (8, 12, 6, 20)]
    recs = make_set(rng, ASCII, pats, [2] * 4, True, extra=6)[:10 if small else 24] + [b"", b"x"]
    for seqs in (recs, tuple(recs), [bytearray(r) for r in recs]):
        for lim in LIMITS:
            assert find_near_matches_batch_in_each(pats, seqs, **lim) == _each(pats, seqs, lim), lim
    resident = DeviceSequenceSet(recs)
    for lim in LIMITS:
        assert find_near_matches_batch_in_each(pats, resident, **lim) == _each(pats, recs, lim), lim
        assert find_near_matches_batch_in_each(pats, resident, **lim) == [
            {r: ms for r, ms in enumerate(find_near_matches_in_each(p, resident, **{
                k: (v[q] if isinstance(v, list) else v) for k, v in lim.items()})) if ms} for q, p in enumerate(pats)]
    resident.close()
    texts = [r.decode("latin-1") for r in recs]
    tpats = [p.decode("latin-1") for p in pats]
    for lim in LIMITS[1:3]:
        assert find_near_matches_batch_in_each(tpats, texts, **lim) == _each(tpats, texts, lim), lim
    # a wide-symbol set, reduced again for each new batch alphabet (its records declared again)
    wide = ["αβγδ" + t + "ωψ" for t in texts] + ["", "γδ€"]
    resident = DeviceSequenceSet(wide)
    for batch_pats in (["γδ" + tpats[0][:3], tpats[1]], ["€αβ", "ψ\U0001F600", tpats[2]], tpats):
        for lim in (dict(max_l_dist=1), dict(max_substitutions=1, max_insertions=0, max_deletions=0)):
            assert find_near_matches_batch_in_each(batch_pats, resident, **lim) == _each(batch_pats, wide, lim)
    # more than 255 distinct symbols over the batch: the patterns go one by one
    many = ["".join(chr(0x400 + 40 * q + j) for j in range(40)) for q in range(7)]
    wide2 = [many[q % 7][5:25] + "xyz" + many[(q + 3) % 7][:12] for q in range(10)]
    resident2 = DeviceSequenceSet(wide2)
    assert find_near_matches_batch_in_each(many, resident2, max_l_dist=1) == _each(many, wide2, dict(max_l_dist=1))
    resident2.close()
    assert find_near_matches_batch_in_each(many, wide2, max_l_dist=2) == _each(many, wide2, dict(max_l_dist=2))
    resident.close()
    # empty inputs and the errors of find_near_matches_batch, raised before anything is uploaded
    assert find_near_matches_batch_in_each([], recs, max_l_dist=1) == []
    assert find_near_matches_batch_in_each(pats, [], max_l_dist=1) == [{} for _ in pats]
    assert find_near_matches_batch_in_each(pats[:1], [b"", b""], max_l_dist=1) == [{}]
    with pytest.raises(ValueError, match="No limitations given!"):
        find_near_matches_batch_in_each(pats, recs)
    with pytest.raises(ValueError, match="No limitations given!"):
        find_near_matches_batch_in_each(pats, [])
    with pytest.raises(ValueError, match="Given subsequence is empty!"):
        find_near_matches_batch_in_each([pats[0], b""], [], max_l_dist=1)
    with pytest.raises(ValueError, match="subsequence must not be empty"):
        find_near_matches_batch_in_each([b""], recs, max_l_dist=0)
    with pytest.raises(ValueError, match="one max_l_dist per subsequence"):
        find_near_matches_batch_in_each(pats, recs, max_l_dist=[1, 2])
    with pytest.raises(TypeError):
        find_near_matches_batch_in_each(pats, b"not a list", max_l_dist=1)
    with pytest.raises(TypeError):
        find_near_matches_batch_in_each(tpats, recs, max_l_dist=1)


def test_golden_records_in_batches_over_a_set(cuda_device, stride=1):
    """The stored find_near_matches calls grouped by their limits, each group one batch over a set of all the golden
    sequences: the entry of each call's own sequence is the single search of it."""
    recs = [r for r in load_golden("ref_suite_calls.json") if r["fn"] == "find_near_matches" and "exc" not in r]
    recs = recs[::stride]
    seqs = sorted(set(bytes.fromhex(r["args"][1]) for r in recs))
    where = {s: i for i, s in enumerate(seqs)}
    groups = {}
    for rec in recs:
        a = rec["args"]
        groups.setdefault(tuple(a[2:6]), []).append((bytes.fromhex(a[0]), bytes.fromhex(a[1])))
    resident = DeviceSequenceSet(seqs)
    for lim, calls in groups.items():
        pats = [p for p, _ in calls if p]
        if not pats:
            continue
        got = find_near_matches_batch_in_each(pats, resident, *lim[3:], max_substitutions=lim[0],
                                              max_insertions=lim[1], max_deletions=lim[2])
        for q, (p, hay) in enumerate((p, h) for p, h in calls if p):
            assert got[q].get(where[hay], []) == find_near_matches(p, hay, *lim), (lim, p, hay)
    resident.close()


def test_demultiplexing_at_full_size(cuda_device):
    """About a million DNA reads of 150 bytes and 96 barcodes of 8..24 bytes with 1..2 substitutions, plus Levenshtein
    barcodes: every pattern's lists on a sample of records equal its find_near_matches_in_each."""
    if EMU:
        pytest.skip("needs a real GPU: a million reads")
    rng = np.random.default_rng(28)
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
    got = find_near_matches_batch_in_each(codes, resident, max_substitutions=subs, max_insertions=0, max_deletions=0)
    sample = set(rng.choice(n, size=20_000, replace=False).tolist())
    for q, c in enumerate(codes):
        each = find_near_matches_in_each(c, resident, max_substitutions=subs[q], max_insertions=0, max_deletions=0)
        assert {r: ms for r, ms in got[q].items()} == {r: ms for r, ms in enumerate(each) if ms}, q
        for r in list(sample)[:200]:
            assert got[q].get(r, []) == find_near_matches(c, reads[r], max_substitutions=subs[q], max_insertions=0,
                                                          max_deletions=0), (q, r)
    lev = codes[:16]
    got = find_near_matches_batch_in_each(lev, resident, max_l_dist=1)
    for q, c in enumerate(lev):
        each = find_near_matches_in_each(c, resident, max_l_dist=1)
        for r in sample:
            assert got[q].get(r, []) == each[r], (q, r)
    resident.close()
