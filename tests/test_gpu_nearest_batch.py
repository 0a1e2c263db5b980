"""fzb_nearest_distance_batch / fzb_nearest_best_per_record, nearest_distance_batch / find_nearest_matches_batch /
nearest_pattern_in_each (DESIGN.md section 5.15): many patterns without a distance limit.  The reference is
`nearest_E` of test_gpu_nearest.py (a numpy restatement of Sellers' table) per pattern, reduced over the patterns by
`reduce_rows`, which states the tie rules: the smallest (dist, index) first, its first end, then the smallest
(dist, index) among the other patterns.  `small` keeps the sizes the CPU emulator replays
(tests/test_emu_nearest_batch.py)."""
import os

import numpy as np
import pytest

from fuzzysearch_b200 import (DeviceSequence, DeviceSequenceSet, NearestDistances, NearestPatterns, _native as F,
                              find_near_matches_batch, find_nearest_matches_batch, nearest_distance,
                              nearest_distance_batch, nearest_distance_in_each, nearest_pattern_in_each)
from test_gpu_nearest import nearest, nearest_rows
from test_gpu_records import joined, rand

pytestmark = pytest.mark.gpu

THREADS, MIN_SEG = 256, 1024  # nearest_kernels.cuh / api.cu (kNearBatchMinSeg)


def sm_count():
    if os.environ.get("FZB_EMU_SMS") and F.lib() is not None and hasattr(F.lib(), "fzb_emu_live_allocations"):
        return int(os.environ["FZB_EMU_SMS"])
    import torch
    return torch.cuda.get_device_properties(0).multi_processor_count


def warp_seg(n, groups, wide=False, sms=None):
    """nearest_batch's bytes per warp (api.cu): one wave of CTAs over all groups of a class"""
    gx = max(1, (sms or sm_count()) * (3 if wide else 4) // groups)
    warps = gx * THREADS // 32
    return max(MIN_SEG, ((n + warps - 1) // warps + 15) // 16 * 16)


def reduce_rows(D, E):
    """(pattern, dist, end, second_pattern, second_dist) of every column of D / E (patterns x records)"""
    D, E = np.asarray(D, dtype=np.int64), np.asarray(E, dtype=np.int64)
    P, R = D.shape
    cols = np.arange(R)
    pat = np.argmin(D, axis=0)  # the first minimum: the smallest index among equal distances
    dist, end = D[pat, cols], E[pat, cols]
    if P == 1:
        return pat, dist, end, np.full(R, -1), np.full(R, -1)
    D2 = D.copy()
    D2[pat, cols] = 1 << 20
    pat2 = np.argmin(D2, axis=0)
    return pat, dist, end, pat2, D2[pat2, cols]


def expected(pats, recs):
    """reduce_rows over nearest() of every (pattern, record)"""
    D = np.array([[nearest(P, r)[0] for r in recs] for P in pats]).reshape(len(pats), len(recs))
    E = np.array([[nearest(P, r)[2] for r in recs] for P in pats]).reshape(len(pats), len(recs))
    return reduce_rows(D, E)


def expected_stacked(pats, recs, pad):
    """the same, the records stacked into one array padded with a byte no pattern holds (such bytes can neither lower
    E nor move its first minimum)"""
    L = max([len(r) for r in recs] + [1])
    rows = np.full((len(recs), L), pad, dtype=np.uint8)
    for i, r in enumerate(recs):
        rows[i, :len(r)] = np.frombuffer(r, dtype=np.uint8)
    DE = [nearest_rows(P, rows) for P in pats]
    return reduce_rows(np.array([d for d, _ in DE]), np.array([e for _, e in DE]))


def check_records(hs, pats, recs, exp=None, ctx=()):
    buf, off = joined(recs)
    hs.upload(buf)
    hs.set_records(off)
    cols, st = hs.nearest_best_per_record(pats)
    assert [c.dtype for c in cols] == [np.int32, np.int32, np.int64, np.int32, np.int32]
    exp = expected(pats, recs) if exp is None else exp
    for name, got, want in zip(("pattern", "dist", "end", "second_pattern", "second_dist"), cols, exp):
        bad = np.flatnonzero(np.asarray(got) != np.asarray(want))
        assert bad.size == 0, (ctx, name, bad[:5], np.asarray(got)[bad[:5]], np.asarray(want)[bad[:5]])
    assert st["route"] == "nearest/batch-bit-vector-scan"
    return cols


def check_whole(hs, pats, S, ctx=()):
    dist, end, st = hs.nearest_distance_batch(pats)
    exp = [nearest(P, S) for P in pats]
    assert dist.tolist() == [e[0] for e in exp], ctx
    assert end.tolist() == [e[2] for e in exp], ctx
    assert st["route"] == "nearest/batch-bit-vector-scan"


def mixed_patterns(rng, alphabet, count, lo=1, hi=64):
    return [rand(rng, alphabet, int(m)) for m in rng.integers(lo, hi + 1, size=count)]


def test_group_geometry(cuda_device, small=False):
    """1 to 200 patterns: partial, full and several groups, both word classes, the fold path for 65-255 symbols, an
    input order unlike the sorted one, and lengths 1-64 inside one group (warm-ups far longer than a lane's own 2m)."""
    rng = np.random.default_rng(31)
    hs = F.Haystack.alloc(1 << 16, device=cuda_device)
    recs = [rand(rng, b"ACGT", int(n)) for n in rng.integers(0, 200 if small else 400, size=40 if small else 120)]
    S = rand(rng, b"ACGT", 3000 if small else 20000)
    for count in (1, 31, 32, 33, 64, 65, 200):
        if small and count in (31, 64):
            continue
        pats = mixed_patterns(rng, b"ACGT", count)
        for r, P in zip(rng.integers(0, len(recs), size=count // 3), pats):  # near copies inside some records
            rec = bytearray(recs[r] + P)
            rec[len(recs[r]) + len(P) // 2:len(recs[r]) + len(P) // 2 + 1] = b"N"
            recs[r] = bytes(rec)
        if count in (33, 65, 200):
            pats[count // 2] = rand(rng, b"ACGT", int(rng.integers(65, 256)))  # the fold path
            pats[-1] = rand(rng, b"ACGT", 100)
        check_records(hs, pats, recs, expected_stacked(pats, recs, ord("x")), (count,))
        hs.set_records(None)
        hs.upload(S)
        check_whole(hs, pats, S, (count,))
    # one group holding lengths 1..32, one holding 33..64, in an order the host has to sort
    pats = [rand(rng, b"ab", m) for m in rng.permutation(np.arange(1, 65)).tolist()]
    recs = [rand(rng, b"ab", int(n)) for n in rng.integers(0, 300, size=60)]
    check_records(hs, pats, recs, expected_stacked(pats, recs, ord("x")))
    hs.set_records(None)
    for n in (0, 1, 63, 129, 2000):
        S = rand(rng, b"ab", n)
        hs.upload(S)
        check_whole(hs, pats, S, (n,))
    hs.close()


def test_ties_empty_records_and_prefill(cuda_device):
    """Equal distances inside one group and across groups, equal ends; empty and 1-byte records; patterns whose d*
    equals m (never reported by a lane) as the winner and as the runner-up."""
    rng = np.random.default_rng(32)
    hs = F.Haystack.alloc(1 << 16, device=cuda_device)
    same = [b"GATTACA"] * 3 + [b"GATTTCA", b"GATTACA"]  # equal patterns: equal (dist, end), the smallest index wins
    across = [rand(rng, b"ACGT", 20) for _ in range(40)] + [b"GATTACA"] + [rand(rng, b"ACGT", 40) for _ in range(40)] \
        + [b"GATTACA"]  # the two copies sit in different groups and classes are mixed
    recs = [b"", b"A", b"C", b"xxGATTACAxxGATTACA", b"GATTCA", b"zzzz", b"", b"GATTACA"[:6]]
    for pats in (same, across):
        check_records(hs, pats, recs)
    # no pattern symbol anywhere: d* = m for all, the prefill alone answers -- the shortest first, then by index
    never = [b"abc", b"ab", b"xy", b"abcd", b"q"]
    check_records(hs, never, [b"", b"\x01", b"ZZZZZZ"])
    # the runner-up never reports: the winner is found, the second is the shortest other pattern at d* = m
    check_records(hs, [b"GATTACA", b"qq", b"qqq", b"TTT"], [b"GATTACA", b"", b"CCCCCC", b"TT"])
    cols = check_records(hs, [b"qq", b"GATTACA"], [b"GATTACA"])
    assert [int(c[0]) for c in cols] == [1, 0, 7, 0, 2]
    # a single pattern: no runner-up; no patterns at all: -1 everywhere
    cols = check_records(hs, [b"GAT"], [b"", b"GAT", b"GT"])
    assert cols[3].tolist() == [-1] * 3 and cols[1].tolist() == [3, 0, 1]
    cols, _ = hs.nearest_best_per_record([])
    assert all(c.tolist() == [-1] * 3 for c in cols)
    hs.set_records(None)
    hs.upload(b"xxGATTACAxxGATTTACA")
    check_whole(hs, same + never, b"xxGATTACAxxGATTTACA")
    assert [len(c) for c in hs.nearest_distance_batch([])[:2]] == [0, 0]
    hs.close()


def test_byte_values(cuda_device):
    """NUL patterns against the separators and the padding; all byte values in patterns and texts."""
    rng = np.random.default_rng(33)
    hs = F.Haystack.alloc(1 << 16, device=cuda_device)
    recs = [b"", b"\0", b"ab", b"\0\0", b"", b"a\0", b"\0a", b"\0" * 5, b""]
    pats = [b"\0", b"\0\0", b"\0\0\0", b"a\0\0a", b"\0" * 40, b"\0" * 70]
    check_records(hs, pats, recs)
    hs.set_records(None)
    for S in (b"abcd" * 33, b"ab\0", b"\0" * 39):
        hs.upload(S)
        check_whole(hs, pats, S)
    every = bytes(range(256))
    pats = [every[i:i + m] for i, m in zip(rng.integers(0, 200, size=70).tolist(), rng.integers(1, 57, size=70).tolist())]
    pats += [every[:255], bytes(reversed(every))[:130]]
    recs = [rand(rng, every, int(n)) for n in rng.integers(0, 300, size=30)] + [every, every[::-1]]
    check_records(hs, pats, recs)
    hs.set_records(None)
    S = rand(rng, every, 5000) + every
    hs.upload(S)
    check_whole(hs, pats, S)
    hs.close()


def test_split_records_and_seams(cuda_device, small=False):
    """A long record among reads, split over many warp segments; the best occurrence of a pattern planted at every
    offset around warp-segment and tile seams; record sets in three orders."""
    rng = np.random.default_rng(34)
    big = (200 << 10) if small else (9 << 20)
    reads = [rand(rng, b"ACGT", 150) for _ in range(200 if small else 2000)]
    pats = mixed_patterns(rng, b"ACGT", 40, 8, 30) + [rand(rng, b"ACGT", 50), rand(rng, b"ACGT", 90)]
    long_rec = bytearray(rand(rng, b"ACGT", big))
    n_total = len(joined(reads[:len(reads) // 2] + [b"x" * big] + reads[len(reads) // 2:])[0])
    seg = warp_seg(n_total, 2)
    lo = len(joined(reads[:len(reads) // 2])[0])
    for k, P in enumerate(pats[:10]):  # the copies end around seams inside the long record
        at = (k + 3) * 8 * seg - lo + int(rng.integers(-2 * len(P), 2 * len(P)))
        if 0 <= at - len(P) and at < big:
            long_rec[at - len(P):at] = P[:len(P) // 2] + b"T" + P[len(P) // 2 + 1:]
    recs = reads[:len(reads) // 2] + [bytes(long_rec)] + reads[len(reads) // 2:]
    hs = F.Haystack.alloc(n_total + (1 << 16), device=cuda_device)
    buf, off = joined(recs)
    hs.upload(buf)
    hs.set_records(off)
    loop = [hs.nearest_per_record(P)[:2] for P in pats]  # (a device loop: the long record is too long for nearest_E)
    exp = reduce_rows(np.array([d for d, _ in loop]), np.array([e for _, e in loop]))
    check_records(hs, pats, recs, exp, ("long",))
    for order in ("up", "down", "shuffled"):
        ls = list(range(0, 301, 1 if not small else 3))
        ls = ls if order == "up" else ls[::-1] if order == "down" else list(rng.permutation(ls))
        rs = [rand(rng, b"ACGT", int(n)) for n in ls]
        check_records(hs, pats[:35], rs, expected_stacked(pats[:35], rs, ord("x")), (order,))
    hs.set_records(None)
    # whole sequence: short texts, where a warp's segment is MIN_SEG bytes, every offset around its seams
    offsets = range(-3, 2 * 24 + 4, 1 if not small else 5)
    for seam in (MIN_SEG, 8 * MIN_SEG):
        for o in offsets:
            P = [rand(rng, b"ab", 24), rand(rng, b"ab", 40)]
            S = bytearray(b"b" * (2 * seam + 100))
            grown = b"".join(bytes([c]) + (b"b" if rng.random() < 0.5 else b"") for c in P[o % 2])
            S[seam + o - len(grown):seam + o] = grown
            assert warp_seg(len(S), 1, o % 2 == 1) == MIN_SEG
            hs.upload(bytes(S))
            check_whole(hs, P + [b"a" * 9], bytes(S), (seam, o))
    hs.close()


def test_one_million_reads_96_barcodes(cuda_device, small=False):
    """Every row equals a device loop of nearest_per_record over the barcodes plus reduce_rows."""
    rng = np.random.default_rng(35)
    count = 3000 if small else 1_000_000
    barcodes = [rand(rng, b"ACGT", int(m)) for m in rng.integers(8, 25, size=96)]
    rows = np.frombuffer(rand(rng, b"ACGT", count * 150), dtype=np.uint8).reshape(count, 150).copy()
    for r in range(0, count, 2):
        b = np.frombuffer(barcodes[r % 96], dtype=np.uint8).copy()
        b[rng.integers(0, len(b), size=int(rng.integers(0, 3)))] = ord("N")
        rows[r, 10:10 + len(b)] = b
    reads = [bytes(r) for r in rows]
    seqset = DeviceSequenceSet(reads, device=cuda_device)
    got = nearest_pattern_in_each(barcodes, seqset)
    assert isinstance(got, NearestPatterns) and len(got) == count
    hay = seqset._seq.haystack
    loop = [hay.nearest_per_record(b)[:2] for b in barcodes]
    exp = reduce_rows(np.array([d for d, _ in loop]), np.array([e for _, e in loop]))
    for name, g, e in zip(("pattern", "dist", "end", "second_pattern", "second_dist"),
                          (got.pattern, got.dist, got.end, got.second_pattern, got.second_dist), exp):
        assert np.array_equal(g, e), name
    sample = rows[:300]
    exp = reduce_rows(*[np.array(x) for x in zip(*[nearest_rows(b, sample) for b in barcodes])])
    assert np.array_equal(got.pattern[:300], exp[0]) and np.array_equal(got.end[:300], exp[2])
    assert got[0] == (int(got.pattern[0]), int(got.dist[0]), int(got.end[0]))
    seqset.close()


def test_four_gib_64_patterns(cuda_device):
    """The whole form over 4 GiB equals fzb_nearest_distance per pattern."""
    rng = np.random.default_rng(36)
    block = np.frombuffer(b"ACGT", dtype=np.uint8)[rng.integers(0, 4, size=1 << 28, dtype=np.uint8)]
    S = np.tile(block, 16)
    pats = [rand(rng, b"ACGT", m) for m in [20] * 24 + [32] * 24 + [64] * 16]
    for k, P in enumerate(pats[::4]):  # near copies past the repeated block's reach, at far-apart places
        at = (k + 1) * (S.size // 17) + k * 977
        v = np.frombuffer(P, dtype=np.uint8).copy()
        v[len(P) // 3] = ord("N")
        S[at:at + len(P)] = v
    hs = F.Haystack.from_host(S, device=cuda_device)
    dist, end, st = hs.nearest_distance_batch(pats)
    single = [hs.nearest_distance(P) for P in pats]
    assert dist.tolist() == [s[0] for s in single] and end.tolist() == [s[2] for s in single]
    assert st["bytes_scanned"] == 2 * S.size  # one scan per word class
    assert max(dist[::4].tolist()) <= 1
    hs.close()


def test_public_api(cuda_device, small=False):
    rng = np.random.default_rng(37)
    n = 20000 if small else 300000
    S = rand(rng, b"ACGT", n)
    pats = [rand(rng, b"ACGT", int(m)) for m in rng.integers(6, 25, size=12)] + [rand(rng, b"ACGT", 80)]
    S = S[:n // 3] + pats[0] + S[n // 3:2 * n // 3] + pats[1][:5] + b"T" + pats[1][6:] + S[2 * n // 3:]
    got = nearest_distance_batch(pats, S)
    assert isinstance(got, NearestDistances) and len(got) == len(pats)
    assert got.dist.tolist() == [nearest_distance(P, S) for P in pats]
    assert [got[i] for i in range(len(pats))] == [nearest(P, S)[::2] for P in pats]
    ds = DeviceSequence(S, device=cuda_device)
    assert nearest_distance_batch(pats, ds).end.tolist() == got.end.tolist()
    searched = pats[:-1]  # (searching the 80-symbol pattern at its large distance is a different test's business)
    dists = got.dist.tolist()[:-1]
    exp = find_near_matches_batch(searched, S, max_l_dist=dists)
    assert all(exp) and find_nearest_matches_batch(searched, S) == exp
    assert find_nearest_matches_batch(searched, ds) == exp
    caps = [max(d - 1, 0) if i % 2 else d + 2 for i, d in enumerate(dists)]
    capped = find_nearest_matches_batch(searched, ds, max_l_dist=caps)
    assert capped == [e if d <= c else [] for e, d, c in zip(exp, dists, caps)]
    assert find_nearest_matches_batch(searched, S, max_l_dist=0) == [e if d == 0 else [] for e, d in zip(exp, dists)]
    ds.close()
    # str (latin-1 and beyond), the wide-symbol fallback (no common byte alphabet), lists of sets
    for pats_s, seq in ((["café", "lait", "au"], "xx cafe au lait, café ou lait xx" * 3),
                        (["ΑΒΓΔ", "ΕΖΗ", "abc"], "αβγδ ΑΒΓΕΖΗΘ \U0001F600 ΑΒΓΔΕΖΗΘ"),
                        (["".join(chr(0x400 + 5 * i + j) for j in range(5)) for i in range(52)],
                         "".join(chr(0x400 + i) for i in range(0, 300, 2)))):  # 260 distinct symbols
        got = nearest_distance_batch(pats_s, seq)
        assert got.dist.tolist() == [nearest_distance(p, seq) for p in pats_s]
        exp = find_near_matches_batch(pats_s, seq, max_l_dist=got.dist.tolist())
        assert find_nearest_matches_batch(pats_s, seq) == exp
        recs = [seq[:k] for k in range(0, len(seq), max(1, len(seq) // 7))]
        np_ = nearest_pattern_in_each(pats_s, recs)
        loop = [nearest_distance_in_each(p, recs) for p in pats_s]
        want = reduce_rows(np.array([x.dist for x in loop]), np.array([x.end for x in loop]))
        assert [c.tolist() for c in (np_.pattern, np_.dist, np_.end, np_.second_pattern, np_.second_dist)] == \
            [np.asarray(c).tolist() for c in want], pats_s[:3]
    recs = [rand(rng, b"ACGT", int(k)) for k in rng.integers(0, 200, size=50)] + [b"", pats[2]]
    got = nearest_pattern_in_each(pats, recs)
    assert [c.tolist() for c in (got.pattern, got.dist, got.end, got.second_pattern, got.second_dist)] == \
        [np.asarray(c).tolist() for c in expected(pats, recs)]
    short = min(range(len(pats)), key=lambda i: (len(pats[i]), i))
    assert got[len(recs) - 2] == (short, len(pats[short]), 0)
    seqset = DeviceSequenceSet(recs, device=cuda_device)
    again = nearest_pattern_in_each(pats, seqset)
    assert again.end.tolist() == got.end.tolist() and again.second_dist.tolist() == got.second_dist.tolist()
    seqset.close()
    assert len(nearest_pattern_in_each(pats, [])) == 0
    none = nearest_pattern_in_each([], [b"AC", b""])
    assert none.pattern.tolist() == [-1, -1] and none.end.tolist() == [-1, -1]
    assert find_nearest_matches_batch([], S) == [] and len(nearest_distance_batch([], S)) == 0
    for call in (lambda: nearest_distance_batch([b"A", b""], b"abc"),
                 lambda: find_nearest_matches_batch([b""], b"abc"),
                 lambda: nearest_pattern_in_each([b"a", b""], [b"abc"]),
                 lambda: find_nearest_matches_batch([b"a"], b"abc", -1),
                 lambda: find_nearest_matches_batch([b"a"], b"abc", [1, 2])):
        with pytest.raises(ValueError):
            call()


def test_searches_around_the_call_and_refusals(cuda_device):
    """Searches before and after the calls behave as if they had not happened; every refusal leaves the handle
    usable."""
    rng = np.random.default_rng(38)
    S = rand(rng, b"ACGT", 5000)
    P = S[1000:1020]
    pats = [P, S[3000:3010], rand(rng, b"ACGT", 70)]
    hs = F.Haystack.from_host(S, device=cuda_device)
    before = hs.search_levenshtein(P, 2)
    b_raw, b_fin = before.triples(F.RAW), before.triples(F.FINAL)
    held = hs.search_levenshtein(P, 1)
    check_whole(hs, pats, S)
    h_raw = held.triples(F.RAW)
    after = hs.search_levenshtein(P, 2)
    assert (after.triples(F.RAW), after.triples(F.FINAL)) == (b_raw, b_fin)
    again = hs.search_levenshtein(P, 1)
    assert again.triples(F.RAW) == h_raw
    for r in (before, held, after, again):
        r.close()

    def still_good():
        check_whole(hs, pats, S)
        res = hs.search_levenshtein(P, 1)
        assert (1000, 1020, 0) in res.triples(F.FINAL)
        res.close()

    for bad, err in (([P], F.UnsupportedError), ([P, b""], ValueError), ([P, b"A" * 256], F.UnsupportedError)):
        with pytest.raises(err):
            hs.nearest_distance_batch(bad, flags=16 if len(bad) == 1 else 0)
    with pytest.raises(F.UnsupportedError):
        hs.nearest_distance_batch([b"A"] * 65536)
    with pytest.raises(ValueError):
        hs.nearest_best_per_record(pats)  # no record set
    still_good()
    hs.set_records(np.array([0, 2500, 5000], dtype=np.uint64))
    with pytest.raises(F.UnsupportedError):
        hs.nearest_distance_batch(pats)  # a record set
    with pytest.raises(F.UnsupportedError):
        hs.nearest_best_per_record(pats, flags=1)
    with pytest.raises(ValueError):
        hs.nearest_best_per_record([P, b""])
    with pytest.raises(F.UnsupportedError):
        hs.nearest_best_per_record([b"A"] * 65536)
    cols, _ = hs.nearest_best_per_record(pats)
    assert (int(cols[0][0]), int(cols[1][0]), int(cols[2][0])) == (0, 0, 1020)
    hs.set_records(None)
    still_good()
    hs.close()
    shard = F.Haystack.from_host(S[:4096], device=cuda_device, buf_lo=0, global_len=5000, own_lo=0, own_hi=2048)
    with pytest.raises(F.UnsupportedError):
        shard.nearest_distance_batch(pats)
    res = shard.search_levenshtein(P, 0)
    assert res.triples(F.RAW) == [(1000, 1020, 0)]
    res.close()
    shard.close()
    world = F.Haystack.from_host(S, device=cuda_device)
    F.comm_init_local([world])
    with pytest.raises(F.UnsupportedError):
        world.nearest_distance_batch(pats)
    world.close()
