"""The six nearest calls under substitutions only (FZB_F_SUBSTITUTIONS_ONLY, substitutions_only=True; DESIGN.md section
5.16).  Every case compares exactly with `hamming_H`, a numpy restatement that counts the mismatches of every window of
the pattern's length and knows nothing of bit slices, segments, warm-ups or prefills (tests/test_host_nearest_hamming.py
checks it against a plain double loop and the oracle).  `small` keeps the sizes the CPU emulator replays
(tests/test_emu_nearest_hamming.py)."""
import numpy as np
import pytest

from fuzzysearch_b200 import (DeviceSequence, DeviceSequenceSet, NearestDistances, NearestPatterns, _native as F,
                              best_match_in_each, find_near_matches, find_near_matches_batch, find_nearest_matches,
                              find_nearest_matches_batch, nearest_distance, nearest_distance_batch,
                              nearest_distance_in_each, nearest_pattern_in_each)
from test_gpu_nearest import nearest
from test_gpu_records import joined, rand

pytestmark = pytest.mark.gpu

SUB = F.F_SUBSTITUTIONS_ONLY
THREADS, MIN_SEG, BATCH_MIN_SEG = 256, 512, 1024  # nearest_kernels.cuh / api.cu
M_SIZES = (1, 2, 7, 31, 32, 33, 63, 64, 65, 128, 192, 255)
NONE32, NONE64 = 0xFFFFFFFF, (1 << 64) - 1


def hamming_H(P, S):
    """H[..., e - m] = the mismatches of P against S[..., e-m:e] for e in m..n (empty when n < m), for one text or a
    stack of equally long texts.  One pass per pattern position."""
    P = np.frombuffer(bytes(P), dtype=np.uint8)
    S = np.frombuffer(bytes(S), dtype=np.uint8) if isinstance(S, (bytes, bytearray)) else np.asarray(S, np.uint8)
    m, n = len(P), S.shape[-1]
    H = np.zeros(S.shape[:-1] + (max(n - m + 1, 0),), dtype=np.int16)
    if n >= m:
        for j in range(m):
            H += S[..., j:j + n - m + 1] != P[j]
    return H


def hamming(P, S):
    """-> (d*, n_ends, first_end) of one text, None without a window"""
    H = hamming_H(P, S)
    if H.size == 0:
        return None
    d = int(H.min())
    at = np.flatnonzero(H == d)
    return d, int(at.size), int(at[0]) + len(P)


def hamming_rows(P, rows):
    """-> (dist, end) arrays for a stack of equally long texts (-1, -1 when they are shorter than P)"""
    H = hamming_H(P, rows)
    if H.shape[-1] == 0:
        return np.full(H.shape[:-1], -1, np.int32), np.full(H.shape[:-1], -1, np.int64)
    return H.min(axis=-1).astype(np.int32), H.argmin(axis=-1).astype(np.int64) + len(P)


def per_record(P, recs):
    got = [hamming(P, r) for r in recs]
    return [-1 if g is None else g[0] for g in got], [-1 if g is None else g[2] for g in got]


def reduce_rows(D, E):
    """(pattern, dist, end, second_pattern, second_dist) of every column of D / E (patterns x records), -1 in D
    meaning "no value": the smallest (dist, index) among the patterns with a value, its end, then the smallest
    (dist, index) among the others with a value."""
    D, E = np.asarray(D, dtype=np.int64), np.asarray(E, dtype=np.int64)
    big = 1 << 20
    Dk = np.where(D < 0, big, D)
    cols = np.arange(D.shape[1])
    pat = np.argmin(Dk, axis=0)
    has = Dk[pat, cols] < big
    dist, end = np.where(has, D[pat, cols], -1), np.where(has, E[pat, cols], -1)
    D2 = Dk.copy()
    D2[pat, cols] = big
    pat2 = np.argmin(D2, axis=0)
    has2 = D2[pat2, cols] < big
    return (np.where(has, pat, -1), dist, end, np.where(has2, pat2, -1), np.where(has2, D2[pat2, cols], -1))


def expected(pats, recs):
    DE = [per_record(P, recs) for P in pats]
    return reduce_rows([d for d, _ in DE], [e for _, e in DE])


def check_handle(hs, P, S, ctx=()):
    d, n_ends, first, st = hs.nearest_distance(P, SUB)
    want = hamming(P, S)
    assert (d, n_ends, first) == ((NONE32, 0, NONE64) if want is None else want), ctx + (len(P), len(S))
    assert st["route"] == "nearest/substitutions-scan" and st["bytes_scanned"] == len(S)
    return want


def check_records(hs, P, recs, ctx=()):
    buf, off = joined(recs)
    hs.upload(buf)
    hs.set_records(off)
    dist, end, st = hs.nearest_per_record(P, SUB)
    assert dist.dtype == np.int32 and end.dtype == np.int64 and len(dist) == len(recs)
    want_d, want_e = per_record(P, recs)
    assert dist.tolist() == want_d, ctx
    assert end.tolist() == want_e, ctx
    assert st["route"] == "nearest/substitutions-scan"
    return dist, end


def check_whole(hs, pats, S, ctx=()):
    dist, end, st = hs.nearest_distance_batch(pats, SUB)
    want = [hamming(P, S) for P in pats]
    assert dist.tolist() == [-1 if w is None else w[0] for w in want], ctx
    assert end.tolist() == [-1 if w is None else w[2] for w in want], ctx
    assert st["route"] == "nearest/substitutions-batch-scan"


def check_batch_records(hs, pats, recs, exp=None, ctx=()):
    buf, off = joined(recs)
    hs.upload(buf)
    hs.set_records(off)
    cols, st = hs.nearest_best_per_record(pats, SUB)
    exp = expected(pats, recs) if exp is None else exp
    for name, got, want in zip(("pattern", "dist", "end", "second_pattern", "second_dist"), cols, exp):
        bad = np.flatnonzero(np.asarray(got) != np.asarray(want))
        assert bad.size == 0, (ctx, name, bad[:5], np.asarray(got)[bad[:5]], np.asarray(want)[bad[:5]])
    assert st["route"] == "nearest/substitutions-batch-scan"
    return cols


def mixed_patterns(rng, alphabet, count, lo=1, hi=64):
    return [rand(rng, alphabet, int(m)) for m in rng.integers(lo, hi + 1, size=count)]


def test_pattern_sizes_and_short_texts(cuda_device, small=False):
    """m = 1..255 over every word-class edge; texts shorter than, as long as and one longer than m."""
    rng = np.random.default_rng(61)
    hs = F.Haystack.alloc(1 << 16, device=cuda_device)
    for m in M_SIZES:
        for alphabet in (b"ab", b"ACGT", bytes(range(256))):
            P = rand(rng, alphabet, m)
            for n in sorted({0, 1, m - 1, m, m + 1, 2 * m + 3, 700}):
                if small and n == 700 and m not in (32, 33, 255):
                    continue
                S = bytearray(rand(rng, alphabet, n))
                if n >= m and rng.random() < 0.5:
                    S[n - m:] = P  # an exact occurrence closing the text
                hs.upload(bytes(S))
                check_handle(hs, P, bytes(S), (alphabet[:4],))
    hs.close()


def test_lengths_around_segments_tiles_and_grid_passes(cuda_device, small=False):
    rng = np.random.default_rng(62)
    tile = THREADS * MIN_SEG
    lengths = [MIN_SEG + d for d in range(-17, 18)] + [tile + d for d in range(-17, 18, 1 if not small else 5)]
    if small:
        passes = 2 * 4 * tile  # FZB_EMU_SMS=2, four CTAs per SM
        lengths += [passes - 1, 2 * passes + 3]
    base = rand(rng, b"ACGT", max(lengths))
    hs = F.Haystack.alloc(max(lengths), device=cuda_device)
    for m in (20, 40):
        P = rand(rng, b"ACGT", m)
        for n in lengths if m == 20 else lengths[::7]:
            S = bytearray(base[:n])
            if n >= m:
                S[n - m:] = P[:m - 1] + b"N"  # the best end is the last position
            hs.upload(bytes(S))
            check_handle(hs, P, bytes(S))
    hs.close()
    if not small:  # 160 MB: several tiles per CTA
        n = 160_000_003
        S = bytearray(rand(rng, b"ACGT", n))
        P = b"GATTACAGGTCCA"
        S[n - 13:] = P
        S[77_000_000:77_000_013] = P
        hs = F.Haystack.from_host(bytes(S), device=cuda_device)
        assert check_handle(hs, P, bytes(S))[0] == 0
        hs.close()


def test_best_window_at_every_offset_around_the_seams(cuda_device, small=False):
    """The single best window ends at every offset around a segment seam and a tile seam; a window that starts up to
    m - 1 bytes before the seam is only found with the full m - 1 bytes of warm-up."""
    rng = np.random.default_rng(63)
    for m, seam, step in ((24, MIN_SEG, 1 if not small else 3), (64, THREADS * MIN_SEG, 1 if not small else 9)):
        hs = F.Haystack.alloc(2 * seam, device=cuda_device)
        for o in range(-4, m + 6, step):
            P = rand(rng, b"ab", m)
            S = bytearray(b"c" * (2 * seam))  # no pattern symbol: every other window is at m
            v = bytearray(P)
            v[m // 2] = ord("c")
            S[seam + o - m:seam + o] = v
            hs.upload(bytes(S))
            assert check_handle(hs, P, bytes(S)) == (1, 1, seam + o), o
        hs.close()


def test_ties_extremes_and_byte_values(cuda_device):
    rng = np.random.default_rng(64)
    hs = F.Haystack.alloc(1 << 16, device=cuda_device)
    cases = [(b"GATTACA", b"xxGATTACAxxGATTACAxxxGATTACA"),            # d* = 0, three ends
             (b"GATTACA", b"xxGATTCCxxGATTTCAxx"),                      # ties at d* = 1
             (b"abc", b"xyzxyzxyz" * 100),                              # d* = m: every window
             (b"\0\0\0\0", b"abcd" * 33),                               # a NUL pattern against the zero padding
             (b"\0\0\0", b"ab\0"), (b"\0" * 40, b"\0" * 39), (b"\0" * 70, b"x" * 127 + b"\0"),
             (bytes(range(128, 160)), rand(rng, bytes(range(120, 170)), 3000)),
             (bytes(range(200, 256)) + bytes(range(9)), bytes(range(256)) * 9),
             (bytes(range(256))[:255], bytes(reversed(range(256))) * 3 + bytes(range(256)))]
    for P, S in cases:
        hs.upload(S)
        check_handle(hs, P, S)
    hs.upload(b"xyzxyzxyz")
    assert hs.nearest_distance(b"abc", SUB)[:3] == (3, 7, 3)
    hs.upload(b"ab")
    assert hs.nearest_distance(b"abc", SUB)[:3] == (NONE32, 0, NONE64)
    assert hs.nearest_distance(b"abc")[:3] == nearest(b"abc", b"ab")  # Levenshtein on the same handle right after
    hs.close()


def test_record_sets(cuda_device, small=False):
    rng = np.random.default_rng(65)
    hs = F.Haystack.alloc(12 << 20, device=cuda_device)
    P = b"GATTACAGATC"
    lengths = list(range(0, 301))
    for order in ("up", "down", "shuffled"):
        ls = lengths if order == "up" else lengths[::-1] if order == "down" else list(rng.permutation(lengths))
        check_records(hs, P, [rand(rng, b"ACGT", int(n)) for n in ls], (order,))
    recs = [b"", b"\0", b"ab", b"\0\0", b"", b"a\0", b"\0a", b"\0" * 5, b""]
    for Pz in (b"\0", b"\0\0", b"\0\0\0", b"a\0\0a", b"\0" * 40):
        check_records(hs, Pz, recs, (Pz,))
    big = (1 << 20) if small else (9 << 20)
    for m in (11, 40, 70):
        Pm = rand(rng, b"ACGT", m)
        long_rec = bytearray(rand(rng, b"ACGT", big))
        long_rec[big - m:] = Pm
        recs = [Pm] + [rand(rng, b"ACGT", 150) for _ in range(40)] + [bytes(long_rec)] + \
               [rand(rng, b"ACGT", 150) for _ in range(40)] + [Pm[:-1]]
        dist, end = check_records(hs, Pm, recs, (m,))
        assert (dist[0], end[0]) == (0, m) and dist[41] == 0 and (dist[-1], end[-1]) == (-1, -1)
        hs.set_records(None)
        for r in (0, 7, 41):
            hs.upload(recs[r])
            assert hs.nearest_distance(Pm, SUB)[::2] == (int(dist[r]), int(end[r]))
    hs.close()


def test_one_million_reads_one_adapter(cuda_device, small=False):
    rng = np.random.default_rng(66)
    count, n = (3000, 150) if small else (1_000_000, 150)
    P = b"AGATCGGAAGAGCACACGTCTGAAC"
    rows = np.frombuffer(rand(rng, b"ACGT", count * n), dtype=np.uint8).reshape(count, n).copy()
    at = rng.integers(0, n - 25, size=count)
    for r in range(0, count, 3):
        v = np.frombuffer(P, dtype=np.uint8).copy()
        v[rng.integers(0, 25, size=int(rng.integers(0, 4)))] = ord("N")
        rows[r, at[r]:at[r] + 25] = v
    got = nearest_distance_in_each(P, [bytes(r) for r in rows], substitutions_only=True)
    assert isinstance(got, NearestDistances) and len(got) == count
    d, e = zip(*[hamming_rows(P, rows[lo:lo + 100_000]) for lo in range(0, count, 100_000)])
    assert np.array_equal(got.dist, np.concatenate(d)) and np.array_equal(got.end, np.concatenate(e))


def test_batch_geometry(cuda_device, small=False):
    """1 to 200 patterns: partial, full and several groups of both word classes, mixed m in one group, the fold for
    65-255 symbols, shuffled order; every row against the single calls."""
    rng = np.random.default_rng(67)
    hs = F.Haystack.alloc(1 << 16, device=cuda_device)
    S = bytearray(rand(rng, b"ACGT", 6000 if not small else 3000))
    recs = [rand(rng, b"ACGT", int(n)) for n in rng.integers(0, 300, size=40)] + [bytes(S[:2500])]
    for count in ((1, 31, 32, 33, 64, 65, 200) if not small else (1, 33, 65)):
        pats = mixed_patterns(rng, b"ACGT", count)
        if count >= 32:
            pats[count // 2] = rand(rng, b"ACGT", 100)  # the fold
            pats[count // 3] = rand(rng, b"ACGT", 255)
        for k, P in enumerate(pats[:6]):
            at = 300 + k * 400
            S[at:at + len(P)] = P[:len(P) // 2] + b"N" + P[len(P) // 2 + 1:]
        hs.set_records(None)
        hs.upload(bytes(S))
        check_whole(hs, pats, bytes(S), (count,))
        if count in (1, 65):
            dist, end, _ = hs.nearest_distance_batch(pats, SUB)
            single = [hs.nearest_distance(P, SUB) for P in pats]
            assert dist.tolist() == [-1 if s[0] == NONE32 else s[0] for s in single]
            assert end.tolist() == [-1 if s[0] == NONE32 else s[2] for s in single]
        check_batch_records(hs, pats, recs, ctx=(count,))
        cols, _ = hs.nearest_best_per_record(pats, SUB)
        loop = [hs.nearest_per_record(P, SUB)[:2] for P in pats]
        want = reduce_rows([d for d, _ in loop], [e for _, e in loop])
        assert all(np.array_equal(c, w) for c, w in zip(cols, want)), count
    hs.close()


def test_batch_patterns_longer_than_records_and_ties(cuda_device):
    """Patterns that do not fit some records, as would-be winners (a long exact copy) and as runner-ups; ties in
    distance between patterns; rows where one or no pattern fits."""
    hs = F.Haystack.alloc(1 << 16, device=cuda_device)
    pats = [b"GATTACAGATTACA", b"ACGT", b"TTTT", b"GATTACAGATTACAGATTACAGATTACAGATTACAGATTACAGATTACAGATTACAGATTACAG"
            b"ATTACAGATTACA"]
    recs = [b"", b"A", b"ACG", b"ACGT", b"TTTA", b"GATTACAGATTACA", pats[3][:70], pats[3], pats[3] + b"TTTT",
            b"xxxxxxxxxxxxxx", b"ACGTTTTT", b"GATTACAGATTAC"]
    cols = check_batch_records(hs, pats, recs)
    assert all(c[:3].tolist() == [-1] * 3 for c in cols)  # no pattern fits "", "A" or "ACG"
    assert [int(c[3]) for c in cols] == [1, 0, 4, 2, 3]  # "ACGT": only ACGT and TTTT fit
    assert cols[0][7] == 0 and cols[3][7] == 3  # a tie at 0 with the 79-symbol copy: the smaller index wins
    hs.set_records(None)
    for S in (b"ACGT", b"GATTACA", b"x" * 100):
        hs.upload(S)
        check_whole(hs, pats, S)
    hs.close()


def test_batch_byte_values_and_seams(cuda_device, small=False):
    rng = np.random.default_rng(68)
    hs = F.Haystack.alloc(1 << 20, device=cuda_device)
    pats = [bytes(rng.integers(0, 256, size=int(m), dtype=np.uint8)) for m in (1, 5, 31, 32, 33, 64, 65, 200)]
    pats += [b"\0" * 3, b"\0a\0"]
    S = bytearray(rng.integers(0, 256, size=40000, dtype=np.uint8).tobytes())
    for k, P in enumerate(pats):
        at = 1000 + 3900 * k
        S[at:at + len(P)] = P
    hs.upload(bytes(S))
    check_whole(hs, pats, bytes(S))
    recs = [bytes(S[i:i + int(n)]) for i, n in zip(range(0, 40000, 1300), rng.integers(0, 400, size=31))]
    recs += [b"", b"\0", b"\0\0\0"]
    check_batch_records(hs, pats, recs)
    # the best window of every pattern of a group ends around a warp's segment seam
    seg = BATCH_MIN_SEG
    for o in range(-3, 40, 1 if not small else 7):
        grp = [rand(rng, b"ab", int(m)) for m in (8, 20, 32)]
        T = bytearray(b"c" * (16 * seg))
        for j, P in enumerate(grp):
            end = (j + 1) * 4 * seg + o
            T[end - len(P):end] = P[:-1] + b"c"
        hs.upload(bytes(T))
        check_whole(hs, grp, bytes(T), (o,))
    hs.close()


def test_one_million_reads_96_barcodes(cuda_device, small=False):
    """Every row equals the loop of per-record calls plus the reduction, and, wherever dist <= 2, the row of
    best_match_in_each(max_substitutions=2, max_insertions=0, max_deletions=0)."""
    rng = np.random.default_rng(69)
    count = 3000 if small else 1_000_000
    barcodes = [rand(rng, b"ACGT", int(m)) for m in rng.integers(8, 25, size=96)]
    rows = np.frombuffer(rand(rng, b"ACGT", count * 150), dtype=np.uint8).reshape(count, 150).copy()
    for r in range(0, count, 2):
        b = np.frombuffer(barcodes[r % 96], dtype=np.uint8).copy()
        b[rng.integers(0, len(b), size=int(rng.integers(0, 4)))] = ord("N")
        rows[r, 10:10 + len(b)] = b
    seqset = DeviceSequenceSet([bytes(r) for r in rows], device=cuda_device)
    got = nearest_pattern_in_each(barcodes, seqset, substitutions_only=True)
    assert isinstance(got, NearestPatterns) and len(got) == count
    hay = seqset._seq.haystack
    loop = [hay.nearest_per_record(b, SUB)[:2] for b in barcodes]
    exp = reduce_rows(np.array([d for d, _ in loop]), np.array([e for _, e in loop]))
    for name, g, e in zip(("pattern", "dist", "end", "second_pattern", "second_dist"),
                          (got.pattern, got.dist, got.end, got.second_pattern, got.second_dist), exp):
        assert np.array_equal(g, e), name
    sample = rows[:300]
    exp = reduce_rows(*[np.array(x) for x in zip(*[hamming_rows(b, sample) for b in barcodes])])
    assert all(np.array_equal(g[:300], e) for g, e in
               zip((got.pattern, got.dist, got.end, got.second_pattern, got.second_dist), exp))
    best = best_match_in_each(barcodes, seqset, max_substitutions=2, max_insertions=0, max_deletions=0)
    near = got.dist <= 2
    assert np.array_equal(best.pattern >= 0, near)
    assert np.array_equal(best.pattern[near], got.pattern[near]) and np.array_equal(best.dist[near], got.dist[near])
    assert np.array_equal(best.end[near], got.end[near])
    both = near & (got.second_dist >= 0) & (got.second_dist <= 2)
    assert np.array_equal(best.second_pattern[both], got.second_pattern[both])
    assert np.array_equal(best.second_dist[both], got.second_dist[both])
    seqset.close()


def test_four_gib_64_patterns(cuda_device):
    """The whole form over 4 GiB equals fzb_nearest_distance per pattern."""
    rng = np.random.default_rng(70)
    block = np.frombuffer(b"ACGT", dtype=np.uint8)[rng.integers(0, 4, size=1 << 28, dtype=np.uint8)]
    S = np.tile(block, 16)
    pats = [rand(rng, b"ACGT", m) for m in [20] * 24 + [32] * 24 + [64] * 16]
    for k, P in enumerate(pats[::4]):
        at = (k + 1) * (S.size // 17) + k * 977
        v = np.frombuffer(P, dtype=np.uint8).copy()
        v[len(P) // 3] = ord("N")
        S[at:at + len(P)] = v
    hs = F.Haystack.from_host(S, device=cuda_device)
    dist, end, st = hs.nearest_distance_batch(pats, SUB)
    single = [hs.nearest_distance(P, SUB) for P in pats]
    assert dist.tolist() == [s[0] for s in single] and end.tolist() == [s[2] for s in single]
    assert st["bytes_scanned"] == 2 * S.size
    assert max(dist[::4].tolist()) <= 1
    hs.close()


def test_public_api(cuda_device, small=False):
    rng = np.random.default_rng(71)
    n = 20000 if small else 300000
    S = bytearray(rand(rng, b"ACGT", n))
    P = rand(rng, b"ACGT", 30)
    kw = dict(max_insertions=0, max_deletions=0)
    for planted, pat in ((P, P), (P[:7] + b"T" + P[8:19] + b"N" + P[20:], P), (b"", rand(rng, b"ACGT", 12))):
        S2 = bytes(S[:n // 2] + planted + S[n // 2:])
        d, n_ends, first = hamming(pat, S2)
        assert nearest_distance(pat, S2, substitutions_only=True) == d
        exp = find_near_matches(pat, S2, max_substitutions=d, **kw)
        assert len(exp) == n_ends and exp[0].end == first and exp[0].start == first - len(pat)
        assert find_nearest_matches(pat, S2, substitutions_only=True) == exp
        assert find_nearest_matches(pat, S2, d, substitutions_only=True) == exp
        if d:
            assert find_nearest_matches(pat, S2, d - 1, substitutions_only=True) == []
            assert find_near_matches(pat, S2, max_substitutions=d - 1, **kw) == []
        ds = DeviceSequence(S2, device=cuda_device)
        assert find_nearest_matches(pat, ds, substitutions_only=True) == exp
        assert nearest_distance(pat, ds, substitutions_only=True) == d
        ds.close()
    assert nearest_distance(b"ACGTACGT", b"ACG", substitutions_only=True) is None
    assert find_nearest_matches(b"ACGTACGT", b"ACG", substitutions_only=True) == []
    # str (latin-1, general Unicode: the alphabet reduction keeps symbol equality) and lists of items
    for pat, seq in (("café au lait", "xx cafe au lait, café ou lait xx" * 3),
                     ("ΑΒΓΔΕΖΗΘ", "αβγδ ΑΒΓΕΖΗΘ \U0001F600 ΑΒΓΔΕΖΗΘ"[:-2] + "λ"),
                     ("abc", "ΑΒΓ" * 10),
                     (["x", 3, "y", 4.5], [1, "x", 3, "z", 4.5, (), "x", "y"] * 4)):
        d = nearest_distance(pat, seq, substitutions_only=True)
        exp = find_near_matches(pat, seq, max_substitutions=d, **kw)
        assert exp and find_nearest_matches(pat, seq, substitutions_only=True) == exp, pat
        assert d == 0 or find_near_matches(pat, seq, max_substitutions=d - 1, **kw) == []
    # batches: str, resident, caps, the wide-symbol fallback (no common byte alphabet)
    pats = [rand(rng, b"ACGT", int(m)) for m in rng.integers(6, 25, size=12)] + [rand(rng, b"ACGT", 80)]
    T = bytes(S[:n // 3]) + pats[0] + bytes(S[n // 3:]) + pats[1][:5] + b"N" + pats[1][6:]
    got = nearest_distance_batch(pats, T, substitutions_only=True)
    assert got.dist.tolist() == [nearest_distance(p, T, substitutions_only=True) for p in pats]
    searched, dists = pats[:-1], got.dist.tolist()[:-1]
    exp = find_near_matches_batch(searched, T, max_substitutions=dists, **kw)
    assert all(exp) and find_nearest_matches_batch(searched, T, substitutions_only=True) == exp
    assert [len(e) for e in exp] == [hamming(p, T)[1] for p in searched]
    ds = DeviceSequence(T, device=cuda_device)
    assert find_nearest_matches_batch(searched, ds, substitutions_only=True) == exp
    caps = [max(d - 1, 0) if i % 2 else d + 2 for i, d in enumerate(dists)]
    assert find_nearest_matches_batch(searched, ds, caps, substitutions_only=True) == \
        [e if d <= c else [] for e, d, c in zip(exp, dists, caps)]
    ds.close()
    assert find_nearest_matches_batch([b"ACGTACGT", pats[0]], b"ACG", substitutions_only=True)[0] == []
    assert nearest_distance_batch([b"ACGTACGT"], b"ACG", substitutions_only=True)[0] == (-1, -1)
    for pats_s, seq in ((["café", "lait", "au"], "xx cafe au lait, café ou lait xx" * 3),
                        (["".join(chr(0x400 + 5 * i + j) for j in range(5)) for i in range(52)],
                         "".join(chr(0x400 + i) for i in range(0, 300, 2)))):  # 260 distinct symbols
        got = nearest_distance_batch(pats_s + ["x" * 200], seq, substitutions_only=True)
        assert got.dist.tolist()[:-1] == [nearest_distance(p, seq, substitutions_only=True) for p in pats_s]
        assert got[len(pats_s)] == (-1, -1)
        exp = find_near_matches_batch(pats_s, seq, max_substitutions=got.dist.tolist()[:-1], **kw)
        assert find_nearest_matches_batch(pats_s, seq, substitutions_only=True) == exp
        recs = [seq[:k] for k in range(0, len(seq), max(1, len(seq) // 7))]
        np_ = nearest_pattern_in_each(pats_s, recs, substitutions_only=True)
        loop = [nearest_distance_in_each(p, recs, substitutions_only=True) for p in pats_s]
        want = reduce_rows(np.array([x.dist for x in loop]), np.array([x.end for x in loop]))
        assert [c.tolist() for c in (np_.pattern, np_.dist, np_.end, np_.second_pattern, np_.second_dist)] == \
            [np.asarray(c).tolist() for c in want], pats_s[:3]
    # sets: lists and resident sets; the Levenshtein answers unchanged
    recs = [rand(rng, b"ACGT", int(k)) for k in rng.integers(0, 200, size=50)] + [b"", P]
    got = nearest_distance_in_each(P, recs, substitutions_only=True)
    assert (got.dist.tolist(), got.end.tolist()) == per_record(P, recs)
    assert got[len(recs) - 2] == (-1, -1) and got[len(recs) - 1] == (0, 30)
    seqset = DeviceSequenceSet(recs, device=cuda_device)
    got = nearest_pattern_in_each(pats, seqset, substitutions_only=True)
    assert [c.tolist() for c in (got.pattern, got.dist, got.end, got.second_pattern, got.second_dist)] == \
        [np.asarray(c).tolist() for c in expected(pats, recs)]
    lev = nearest_distance_in_each(P, seqset)
    assert lev.dist.tolist() == [nearest(P, r)[0] for r in recs]
    seqset.close()
    words = ["naïve", "", "ΑΒΓ naive", "nave", "\U0001F600naïv"]
    got = nearest_distance_in_each("naïve", words, substitutions_only=True)
    assert got.dist.tolist() == [0, -1, 1, -1, 5] and got.end.tolist() == [5, -1, 9, -1, 5]


def test_searches_around_the_call_and_refusals(cuda_device):
    """Searches before and after the calls behave as if they had not happened; every other flag, alone or with the
    new one, more than 65 535 patterns, shards and worlds are refused and leave the handle usable."""
    rng = np.random.default_rng(72)
    S = rand(rng, b"ACGT", 5000)
    P = S[1000:1020]
    pats = [P, S[3000:3010], rand(rng, b"ACGT", 70)]
    hs = F.Haystack.from_host(S, device=cuda_device)
    lev_before = hs.nearest_distance(P)[:3], hs.nearest_distance_batch(pats)[:2]
    before = hs.search_hamming(P, 3)
    b_raw = before.triples(F.RAW)
    held = hs.search_levenshtein(P, 1)
    check_handle(hs, P, S)
    check_whole(hs, pats, S)
    h_raw = held.triples(F.RAW)
    after, again = hs.search_hamming(P, 3), hs.search_levenshtein(P, 1)
    assert after.triples(F.RAW) == b_raw and again.triples(F.RAW) == h_raw
    for r in (before, held, after, again):
        r.close()
    lev_after = hs.nearest_distance(P)[:3], hs.nearest_distance_batch(pats)[:2]
    assert lev_after[0] == lev_before[0] and all(np.array_equal(a, b) for a, b in zip(lev_after[1], lev_before[1]))

    def still_good():
        check_handle(hs, P, S)
        check_whole(hs, pats, S)
        res = hs.search_hamming(P, 1)
        assert (1000, 1020, 0) in res.triples(F.FINAL)
        res.close()

    for other in (1, 2, 4, 8, 16, 32, 64, 128, 512):
        for flags in (other, other | SUB):
            with pytest.raises(F.UnsupportedError):
                hs.nearest_distance(P, flags)
            with pytest.raises(F.UnsupportedError):
                hs.nearest_distance_batch(pats, flags)
    with pytest.raises(F.UnsupportedError):
        hs.nearest_distance_batch([b"A"] * 65536, SUB)
    with pytest.raises(ValueError):
        hs.nearest_best_per_record(pats, SUB)  # no record set
    still_good()
    hs.set_records(np.array([0, 2500, 5000], dtype=np.uint64))
    with pytest.raises(F.UnsupportedError):
        hs.nearest_distance(P, SUB)  # a record set
    for other in (1, 16, 128):
        with pytest.raises(F.UnsupportedError):
            hs.nearest_per_record(P, other | SUB)
        with pytest.raises(F.UnsupportedError):
            hs.nearest_best_per_record(pats, other | SUB)
    with pytest.raises(F.UnsupportedError):
        hs.nearest_best_per_record([b"A"] * 65536, SUB)
    dist, end, _ = hs.nearest_per_record(P, SUB)
    second = hamming(P, S[2500:4999])
    assert (dist.tolist(), end.tolist()) == ([0, second[0]], [1020, second[2]])
    hs.set_records(None)
    still_good()
    hs.close()
    shard = F.Haystack.from_host(S[:4096], device=cuda_device, buf_lo=0, global_len=5000, own_lo=0, own_hi=2048)
    with pytest.raises(F.UnsupportedError):
        shard.nearest_distance(P, SUB)
    with pytest.raises(F.UnsupportedError):
        shard.nearest_distance_batch(pats, SUB)
    shard.close()
    world = F.Haystack.from_host(S, device=cuda_device)
    F.comm_init_local([world])
    with pytest.raises(F.UnsupportedError):
        world.nearest_distance(P, SUB)
    with pytest.raises(F.UnsupportedError):
        world.nearest_distance_batch(pats, SUB)
    world.close()
