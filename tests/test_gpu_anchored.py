"""The anchored nearest calls (FZB_F_ANCHOR_START / FZB_F_ANCHOR_END, anchor='start' / 'end'; DESIGN.md section 5.18).
Every case compares exactly with `anchored`, a numpy restatement that builds the prefix-anchored table a pattern row
at a time (D[0][j] = j) and knows nothing of bit vectors, lane groups, early stops, prefills or mirrored walks
(tests/test_host_anchored.py checks it against a plain triple loop and the mirror identity).  `small` keeps the sizes
the CPU emulator replays (tests/test_emu_anchored.py)."""
import numpy as np
import pytest

from fuzzysearch_b200 import (DeviceSequenceSet, NearestDistances, NearestPatterns, _native as F, align_in_each,
                              find_near_matches, nearest_distance_in_each, nearest_pattern_in_each)
from conftest import needs_real_gpu
from test_gpu_records import joined, rand

pytestmark = pytest.mark.gpu

SUB, START, END = F.F_SUBSTITUTIONS_ONLY, F.F_ANCHOR_START, F.F_ANCHOR_END
M_SIZES = (1, 2, 7, 31, 32, 33, 63, 64, 65, 100, 128, 129, 192, 193, 255)


def prefix_row(P, R):
    """A[e] = lev(P, R[0:e]) for e in 0..n: the bottom row of the table with D[i][0] = i and D[0][j] = j, one pattern
    row at a time (the left neighbour through a running minimum)."""
    P = np.frombuffer(bytes(P), dtype=np.uint8)
    R = np.frombuffer(bytes(R), dtype=np.uint8)
    n = len(R)
    idx = np.arange(n + 1, dtype=np.int64)
    row = idx.copy()
    for i, c in enumerate(P, 1):
        t = np.minimum(row[:-1] + (R != c), row[1:] + 1)
        row = np.minimum.accumulate(np.concatenate(([i], t)) - idx) + idx
    return row


def anchored(P, R, anchor, subs=False):
    """-> (dist, start, end) of the anchored nearest match of P in R, None without one (substitutions only, R
    shorter than P).  Ties: the smallest end under 'start', the largest start under 'end'."""
    m, n = len(P), len(R)
    if subs:
        if n < m:
            return None
        w = R[:m] if anchor == "start" else R[n - m:]
        d = int(np.count_nonzero(np.frombuffer(bytes(P), np.uint8) != np.frombuffer(bytes(w), np.uint8)))
        return (d, 0, m) if anchor == "start" else (d, n - m, n)
    if anchor == "start":
        A = prefix_row(P, R)
        e = int(np.argmin(A))
        return int(A[e]), 0, e
    B = prefix_row(bytes(P)[::-1], bytes(R)[::-1])  # B[n - s] = lev(P, R[s:n])
    e = int(np.argmin(B))
    return int(B[e]), n - e, n


def symbols_read(P, R, anchor, subs=False):
    """The symbols the kernel reads of R for P: m under substitutions only (0 without a window), else up to the first
    e with e - m >= the best so far, at most min(n, 2m)."""
    m, n = len(P), len(R)
    if subs:
        return m if n >= m else 0
    A = prefix_row(P, R) if anchor == "start" else prefix_row(bytes(P)[::-1], bytes(R)[::-1])
    best, e = m, 0
    while e < min(n, 2 * m) and e + 1 - m < best:
        e += 1
        best = min(best, int(A[e]))
    return e


def per_record(P, recs, anchor, subs=False):
    """-> (dist, pos) lists as fzb_nearest_per_record returns them: pos the end ('start') or the start ('end')"""
    got = [anchored(P, r, anchor, subs) for r in recs]
    return ([-1 if g is None else g[0] for g in got],
            [-1 if g is None else (g[2] if anchor == "start" else g[1]) for g in got])


def reduce_patterns(pats, recs, anchor, subs=False):
    """-> the columns of fzb_nearest_best_per_record (pattern, dist, pos, second_pattern, second_dist): the smallest
    (dist, index), its pos, and the smallest (dist, index) over the other patterns; -1 where nothing takes part."""
    cols = [[], [], [], [], []]
    for R in recs:
        got = sorted((g[0], i, g) for i, P in enumerate(pats) for g in [anchored(P, R, anchor, subs)] if g is not None)
        if not got:
            row = (-1, -1, -1, -1, -1)
        else:
            d, i, g = got[0]
            pos = g[2] if anchor == "start" else g[1]
            rest = [x for x in got[1:] if x[1] != i]
            row = (i, d, pos) + ((rest[0][1], rest[0][0]) if rest else (-1, -1))
        for c, v in zip(cols, row):
            c.append(v)
    return cols


def flags_of(anchor, subs):
    return (START if anchor == "start" else END) | (SUB if subs else 0)


def set_records(hs, recs):
    buf, off = joined(recs)
    hs.upload(buf)
    hs.set_records(off)


def check_records(hs, P, recs, anchor, subs, ctx=()):
    set_records(hs, recs)
    dist, pos, st = hs.nearest_per_record(P, flags_of(anchor, subs))
    exp = per_record(P, recs, anchor, subs)
    assert dist.tolist() == exp[0], (ctx, P, anchor, subs)
    assert pos.tolist() == exp[1], (ctx, P, anchor, subs)
    assert st["route"] == "nearest/anchored"
    assert st["bytes_scanned"] == sum(symbols_read(P, r, anchor, subs) for r in recs), (ctx, P, anchor, subs)


def check_batch(hs, pats, recs, anchor, subs, ctx=()):
    set_records(hs, recs)
    cols, st = hs.nearest_best_per_record(pats, flags_of(anchor, subs))
    exp = reduce_patterns(pats, recs, anchor, subs)
    for name, got, want in zip(("pattern", "dist", "pos", "second_pattern", "second_dist"), cols, exp):
        assert got.tolist() == want, (ctx, name, len(pats), anchor, subs)
    assert st["route"] == "nearest/anchored"


def mixed_patterns(rng, alphabet, count, lo=1, hi=24):
    return [rand(rng, alphabet, int(n)) for n in rng.integers(lo, hi + 1, size=count)]


BOTH = [(a, s) for a in ("start", "end") for s in (False, True)]


def test_pattern_sizes_and_record_lengths(cuda_device, small=False):
    """m = 1 ... 255 (one word of 32 and 64 bits, every multi-word size), records of 0 ... 300 symbols in three
    orders, shorter than m and 2m, with planted mutated copies at either end."""
    rng = np.random.default_rng(11)
    hs = F.Haystack.alloc(1 << 20)
    sizes = M_SIZES if not small else (1, 7, 32, 33, 64, 65, 130)
    for m in sizes:
        P = rand(rng, b"ACGT", m)
        lengths = list(range(0, 301, 1 if not small else 23)) + [m - 1, m, m + 1, 2 * m - 1, 2 * m, 2 * m + 1]
        lengths = [x for x in lengths if x >= 0]
        recs = []
        for k, n in enumerate(lengths):
            R = bytearray(rand(rng, b"ACGT", n))
            V = bytearray(P)
            for _ in range(int(rng.integers(0, 3))):
                V[int(rng.integers(0, m))] = ord("ACGT"[int(rng.integers(0, 4))])
            if k % 3 == 0 and n >= m:
                R[:m] = V
            elif k % 3 == 1 and n >= m:
                R[n - m:] = V
            recs.append(bytes(R))
        for order in (recs, recs[::-1], [recs[i] for i in rng.permutation(len(recs))]):
            for anchor, subs in BOTH:
                check_records(hs, P, order, anchor, subs, ("m", m))
    hs.close()


def test_lane_groups_and_cta_rows(cuda_device, small=False):
    """G = 1, 2, 4, ..., 32 patterns per record (pattern counts that leave idle lanes), 33, 65 and 1 000 patterns
    (several CTA rows), patterns of both word classes and of more than 64 symbols in one call."""
    rng = np.random.default_rng(12)
    recs = [rand(rng, b"ACGT", int(n)) for n in rng.integers(0, 160, size=300 if not small else 40)]
    counts = (1, 2, 3, 4, 5, 8, 13, 16, 31, 32, 33, 65, 1000) if not small else (1, 3, 8, 33)
    hs = F.Haystack.alloc(len(joined(recs)[0]))
    for count in counts:
        pats = mixed_patterns(rng, b"ACGT", count, 1, 64 if count < 100 else 24)
        for i, P in enumerate(pats[:len(recs)]):  # plant some of them
            r = recs[(7 * i) % len(recs)]
            if len(r) >= len(P):
                recs[(7 * i) % len(recs)] = P + r[len(P):] if i % 2 else r[:len(r) - len(P)] + P
        for anchor, subs in BOTH:
            check_batch(hs, pats, recs, anchor, subs, ("count", count))
    long = pats[:3] + [rand(rng, b"ACGT", 100), rand(rng, b"ACGT", 200)]
    for anchor, subs in BOTH:
        check_batch(hs, long, recs, anchor, subs, "long")
    hs.close()


def test_ties_extremes_separators_and_byte_values(cuda_device):
    """Ties on the end and on the start, dist 0 and dist m, NUL patterns against the separators, all byte values."""
    hs = F.Haystack.alloc(1 << 16)
    recs = [b"", b"A", b"AA", b"AAA", b"ABA", b"AXXA", b"XA", b"AX", b"\0", b"\0\0\0"]
    for P in (b"A", b"AA", b"AXA", b"\0", b"\0\0", b"X" * 5):
        for anchor, subs in BOTH:
            check_records(hs, P, recs, anchor, subs, "ties")
        check_batch(hs, [P, b"A", b"\0"], recs, "start", False, "ties")
        check_batch(hs, [P, b"A", b"\0"], recs, "end", True, "ties")
    rng = np.random.default_rng(13)
    allbytes = bytes(range(256))
    recs = [bytes(rng.permutation(256).astype(np.uint8)[:int(n)]) for n in rng.integers(0, 256, size=50)]
    recs += [allbytes, allbytes[::-1]]
    for P in (allbytes[:64], allbytes[200:], allbytes[:255], bytes(rng.integers(0, 256, 40).astype(np.uint8))):
        for anchor, subs in BOTH:
            check_records(hs, P, recs, anchor, subs, "bytes")
    for anchor, subs in BOTH:
        check_batch(hs, [allbytes[i:i + 20] for i in range(0, 236, 7)], recs, anchor, subs, "bytes")
    hs.close()


def test_long_record_among_reads_and_mirror_identity(cuda_device, small=False):
    """A 9 MiB record among reads costs 2m symbols; 'end' on (P, R) is 'start' on the reversed pair."""
    rng = np.random.default_rng(14)
    big = bytearray(rand(rng, b"ACGT", (9 << 20) if not small else 5000))
    P = rand(rng, b"ACGT", 20)
    big[:20], big[-20:] = P, P
    recs = [rand(rng, b"ACGT", int(n)) for n in rng.integers(0, 150, size=200)]
    recs.insert(77, bytes(big))
    hs = F.Haystack.alloc(len(joined(recs)[0]))
    for anchor, subs in BOTH:
        check_records(hs, P, recs, anchor, subs, "big")
    set_records(hs, recs)
    d_end, s_end, _ = hs.nearest_per_record(P, END)
    set_records(hs, [r[::-1] for r in recs])
    d_start, e_start, _ = hs.nearest_per_record(P[::-1], START)
    n = np.array([len(r) for r in recs])
    assert d_end.tolist() == d_start.tolist()
    assert s_end.tolist() == (n - e_start).tolist()
    assert int(d_end[77]) == 0 and int(s_end[77]) == len(big) - 20
    hs.close()


def test_anchored_against_unanchored(cuda_device, small=False):
    """The anchored dist is at least the unanchored one, and equal where the best unanchored match starts at 0."""
    rng = np.random.default_rng(15)
    P = rand(rng, b"ACGT", 12)
    recs = [rand(rng, b"ACGT", int(n)) for n in rng.integers(0, 80, size=500 if not small else 60)]
    recs = [P[:int(rng.integers(0, 13))] + r if i % 2 else r for i, r in enumerate(recs)]
    free = nearest_distance_in_each(P, recs)
    anch = nearest_distance_in_each(P, recs, anchor="start")
    assert (anch.dist >= free.dist).all()
    for r, R in enumerate(recs):
        ms = find_near_matches(P, R, max_l_dist=int(free.dist[r])) if len(R) else []
        if any(x.start == 0 and x.dist == free.dist[r] for x in ms):
            assert anch.dist[r] == free.dist[r], r


def test_public_api_and_align(cuda_device, small=False):
    """nearest_distance_in_each / nearest_pattern_in_each with anchor=, str and wide-symbol sets, resident and
    uploaded, and align_in_each on the anchored rows (start 0 under 'start', cost = dist)."""
    rng = np.random.default_rng(16)
    pats = [rand(rng, b"ACGT", int(n)) for n in rng.integers(6, 20, size=24)]
    reads = []
    for i in range(400 if not small else 50):
        P = bytearray(pats[i % len(pats)])
        P[int(rng.integers(0, len(P)))] = ord("ACGT"[int(rng.integers(0, 4))])
        tail = rand(rng, b"ACGT", int(rng.integers(0, 60)))
        reads.append(bytes(P) + tail if i % 2 else tail + bytes(P))
    reads += [b"", b"A"]
    for anchor in ("start", "end"):
        for subs in (False, True):
            for seqs in (reads, DeviceSequenceSet(reads)):
                got = nearest_distance_in_each(pats[0], seqs, substitutions_only=subs, anchor=anchor)
                assert isinstance(got, NearestDistances) and got.start is not None
                for r, R in enumerate(reads):
                    exp = anchored(pats[0], R, anchor, subs)
                    assert (int(got.dist[r]), int(got.start[r]), int(got.end[r])) == (exp or (-1, -1, -1)), r
                rows = nearest_pattern_in_each(pats, seqs, substitutions_only=subs, anchor=anchor)
                assert isinstance(rows, NearestPatterns)
                exp = reduce_patterns(pats, reads, anchor, subs)
                assert rows.pattern.tolist() == exp[0] and rows.dist.tolist() == exp[1]
                assert rows.second_pattern.tolist() == exp[3] and rows.second_dist.tolist() == exp[4]
                for r, R in enumerate(reads):
                    if rows.pattern[r] < 0:
                        assert rows.start[r] == -1 and rows.end[r] == -1
                        continue
                    g = anchored(pats[rows.pattern[r]], R, anchor, subs)
                    assert (int(rows.start[r]), int(rows.end[r])) == g[1:], r
                al = align_in_each(pats, seqs, rows, substitutions_only=subs)
                live = rows.pattern >= 0
                assert (al.dist[live] == rows.dist[live]).all()
                assert (al.start[live] == rows.start[live]).all() and (al.end[live] == rows.end[live]).all()
                if anchor == "start":
                    assert (al.start[live] == 0).all()
                if isinstance(seqs, DeviceSequenceSet):
                    seqs.close()
    # str and wide symbols (a pattern alphabet beyond one byte)
    words = ["héllo wörld", "wörld héllo", "", "h€llo", "xx héllo"]
    for anchor in ("start", "end"):
        got = nearest_distance_in_each("héllo", words, anchor=anchor)
        for r, R in enumerate(words):
            exp = anchored(tuple_bytes("héllo", R)[0], tuple_bytes("héllo", R)[1], anchor)
            assert (int(got.dist[r]), int(got.start[r]), int(got.end[r])) == exp, (anchor, r)
        rows = nearest_pattern_in_each(["héllo", "wörld", "€"], words, anchor=anchor)
        assert rows.start is not None and (rows.pattern >= 0).all()
    with pytest.raises(ValueError):
        nearest_distance_in_each(b"AC", [b"ACGT"], anchor="middle")
    with pytest.raises(ValueError):
        nearest_pattern_in_each([b"AC"], [b"ACGT"], anchor=0)
    assert nearest_distance_in_each(b"AC", [b"ACGT"]).start is None
    assert nearest_pattern_in_each([b"AC"], [b"ACGT"]).start is None


def tuple_bytes(P, R):
    """A str pattern and text as one-symbol-per-byte strings over a shared code, for the restatement"""
    code = {c: i + 1 for i, c in enumerate(sorted(set(P) | set(R)))}
    return bytes(code[c] for c in P), bytes(code[c] for c in R)


def test_one_million_reads_96_barcodes(cuda_device, small=False):
    """The demultiplexing workload: reads starting with one of 96 barcodes of 8-24 symbols plus 0-2 edits."""
    rng = np.random.default_rng(17)
    n = 1_000_000 if not small else 300
    codes = [rand(rng, b"ACGT", int(m)) for m in rng.integers(8, 25, size=96)]
    truth = rng.integers(0, 96, size=n)
    reads = []
    for i in range(n):
        b = bytearray(codes[truth[i]])
        for _ in range(int(rng.integers(0, 3))):
            b[int(rng.integers(0, len(b)))] = ord("ACGT"[int(rng.integers(0, 4))])
        reads.append(bytes(b) + rand(rng, b"ACGT", 150 - len(b)))
    hs = F.Haystack.alloc(len(joined(reads)[0]))
    check_at = rng.choice(n, size=min(n, 2000), replace=False)
    for anchor, subs in BOTH:
        set_records(hs, reads)
        cols, _ = hs.nearest_best_per_record(codes, flags_of(anchor, subs))
        sub = [reads[i] for i in check_at]
        exp = reduce_patterns(codes, sub, anchor, subs)
        for got, want in zip(cols, exp):
            assert got[check_at].tolist() == want, (anchor, subs)
    hs.close()


def test_searches_around_the_call_and_refusals(cuda_device):
    """Searches before and after the calls behave as if they had not happened; both anchors together, anchors on the
    whole-sequence calls, any other flag, 65 536 patterns, a record of 2^32 bytes and worlds are refused and leave the
    handle usable."""
    rng = np.random.default_rng(18)
    recs = [rand(rng, b"ACGT", int(n)) for n in rng.integers(0, 100, size=50)]
    P, pats = b"ACGTAC", [b"ACGTAC", b"GGA", rand(rng, b"ACGT", 70)]
    buf, off = joined(recs)
    hs = F.Haystack.from_host(buf, device=cuda_device)
    held = hs.search_levenshtein(P, 1)
    h_raw = held.triples(F.RAW)
    whole = hs.nearest_distance(P)[:3]
    hs.set_records(off)
    exp = {(a, s): (per_record(P, recs, a, s), reduce_patterns(pats, recs, a, s)) for a, s in BOTH}

    def still_good():
        for a, s in BOTH:
            dist, pos, _ = hs.nearest_per_record(P, flags_of(a, s))
            assert [dist.tolist(), pos.tolist()] == list(exp[a, s][0])
            assert [c.tolist() for c in hs.nearest_best_per_record(pats, flags_of(a, s))[0]] == exp[a, s][1]

    still_good()
    assert held.triples(F.RAW) == h_raw  # (the pending result is untouched)
    for s in (0, SUB):
        with pytest.raises(ValueError):
            hs.nearest_per_record(P, START | END | s)
        with pytest.raises(ValueError):
            hs.nearest_best_per_record(pats, START | END | s)
        for other in (1, 16, 128, 512):
            for a in (START, END):
                with pytest.raises(F.UnsupportedError):
                    hs.nearest_per_record(P, other | a | s)
                with pytest.raises(F.UnsupportedError):
                    hs.nearest_best_per_record(pats, other | a | s)
        with pytest.raises(F.UnsupportedError):
            hs.nearest_best_per_record([b"A"] * 65536, START | s)
    still_good()
    hs.set_records(None)
    for fl in (START, END, START | SUB, END | SUB, START | END):
        with pytest.raises(F.UnsupportedError):
            hs.nearest_distance(P, fl)
        with pytest.raises(F.UnsupportedError):
            hs.nearest_distance_batch(pats, fl)
    assert hs.nearest_distance(P)[:3] == whole
    again = hs.search_levenshtein(P, 1)
    assert again.triples(F.RAW) == h_raw
    for r in (held, again):
        r.close()
    hs.close()
    world = F.Haystack.from_host(buf, device=cuda_device)
    F.comm_init_local([world])
    with pytest.raises(F.UnsupportedError):
        world.nearest_distance_batch(pats, START)
    world.close()


def test_records_at_2_32(cuda_device):
    """Record 0 of 2^32 - 1 bytes: 'start' reads its first 2m bytes, 'end' its last (starts past 2^32 come back
    whole); a record of 2^32 bytes is refused and the handle then answers as before."""
    needs_real_gpu("a 4.3 GB record")
    G32 = 1 << 32
    rng = np.random.default_rng(19)
    P = rand(rng, b"ACGT", 24)
    tail = [b"", P + b"ACGT", b"A"]
    off = [0, G32]
    for r in tail:
        off.append(off[-1] + len(r) + 1)
    hs = F.Haystack.alloc(off[-1], device=cuda_device)
    hs.fill_synthetic(b"wxyz", 9)
    for o in off[1:]:
        hs.write(o - 1, b"\0")
    for o, r in zip(off[1:], tail):
        hs.write(o, r)
    hs.write(3, P[:20])
    v = P[:10] + b"A" + P[11:] if P[10:11] != b"A" else P[:10] + b"C" + P[11:]
    hs.write(G32 - 1 - 24, v)
    n0 = G32 - 1
    head, back = hs.read(0, 48), hs.read(n0 - 48, 48)
    hs.set_records(off)
    for anchor, subs in BOTH:
        dist, pos, st = hs.nearest_per_record(P, flags_of(anchor, subs))
        d0 = anchored(P, head if anchor == "start" else back, anchor, subs)
        want0 = (d0[0], d0[2]) if anchor == "start" else (d0[0], d0[1] + n0 - 48)
        exp = per_record(P, tail, anchor, subs)
        assert dist.tolist() == [want0[0]] + exp[0] and pos.tolist() == [want0[1]] + exp[1], (anchor, subs)
        cols, _ = hs.nearest_best_per_record([P, P[:8]], flags_of(anchor, subs))
        want = reduce_patterns([P, P[:8]], [head if anchor == "start" else back] + tail, anchor, subs)
        if anchor == "end":
            want[2][0] += n0 - 48
        assert [c.tolist() for c in cols] == want, (anchor, subs)
    before = hs.nearest_per_record(P, END)[:2]
    hs.set_records([0, G32 + 1] + off[3:])
    for fl in (START, END, START | SUB):
        with pytest.raises(F.UnsupportedError):
            hs.nearest_per_record(P, fl)
        with pytest.raises(F.UnsupportedError):
            hs.nearest_best_per_record([P], fl)
    hs.set_records(off)
    after = hs.nearest_per_record(P, END)[:2]
    assert all(np.array_equal(a, b) for a, b in zip(before, after))
    hs.close()
